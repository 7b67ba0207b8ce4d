"""Static evidence per hot kernel from the built objects (no GPU needed): SASS instruction counts by class
(cuobjdump -sass), registers / spills / shared memory (cuobjdump -res-usage).  Output -> profiles/rNN_sass_summary.txt.

    python tools/sass_summary.py [regex ...]      (default: the kernels of the bench configurations)

UBLKCP = bulk-TMA copies (cp.async.bulk), LDG/STG .256 = 256-bit vector global accesses, IMAD.WIDE = the 32x32+64
multiply-add the limb arithmetic is built on.  Counts are static (one trip of each loop)."""
import glob
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, 'mpyc_b200', 'csrc', '_obj')
DEFAULT = [r'k_split_tiled<2, 1, 3, 0, 1>', r'k_split_tiled<2, 0, 3, 0, 1>', r'k_split_tiled<1, 1, 2, 0, 1>', r'k_split_tiled<4, 1, 4, 0, 1>',
           r'k_split_gen<2, 1, 3, 0, 1, StridedDst>', r'k_recombine_tiled<2, 1, 1, 3>', r'k_recombine_tiled<2, 0, 1, 3>',
           r'k_recombine_tiled<1, 1, 1, 2>', r'k_recombine_tiled<4, 1, 1, 8>', r'k_recombine_tiled<2, 0, 0, 4>', r'k_binop<1, 1, 2, 0, 1>', r'k_binop<1, 0, 2, 0, 1>', r'k_prss_tiles<4, 1, 1, 1, 1>',
           r'k_prss_tiles<4, 1, 1, 1, 0>', r'k_matmul<2, 1', r'k_inv_batch<2, 1>', r'k_prf_reduce<', r'k_gf_split', r'k_gf_recombine',
           # K6, the protocols' raw-value algebra (local.cuh): LDGSTS = cp.async pieces of k_bits_compose
           r'k_bits_compose<2, 1>', r'k_bits_compose<1, 1>', r'k_bits_compose<4, 1>', r'k_bits_decompose<2, 1>', r'k_fma<2, 1, 1, 1>',
           r'k_axpb<2, 1, 1>', r'k_low_bits<2, 1>', r'k_nonzero<2, 1>', r'k_transpose<2>', r'k_scan_cols<2, 1, true>', r'k_binop_rows<2, 1, 1, 1>',
           r'k_conv2d<2, 1>']


def demangle(names):
    out = subprocess.run(['cu++filt'] + names, capture_output=True, text=True).stdout.split('\n')
    res = []
    for nm in out[:len(names)]:
        nm = nm.replace('void ', '')
        nm = nm[:nm.index('>(') + 1] if '>(' in nm else nm.split('(')[0]
        res.append(nm.replace('(int)', '').replace('(bool)', '').replace('true', '1').replace('false', '0'))
    return res


def main():
    pats = sys.argv[1:] or DEFAULT
    rows = []
    for obj in sorted(glob.glob(os.path.join(OBJ, '*.o'))):
        if not obj.endswith(('api.o', 'inst_L1.o', 'inst_L2.o', 'inst_L3.o', 'inst_L4.o', 'inst_layout.o')):
            continue
        sass = subprocess.run(['cuobjdump', '-sass', obj], capture_output=True, text=True).stdout
        res = subprocess.run(['cuobjdump', '-res-usage', obj], capture_output=True, text=True).stdout
        usage = {}
        for mt in re.finditer(r'Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)', res):
            usage[mt.group(1)] = (int(mt.group(2)), int(mt.group(3)), int(mt.group(4)), int(mt.group(5)))
        blocks = sass.split('Function : ')[1:]
        names = [b.split('\n', 1)[0].strip() for b in blocks]
        for name, dem, blk in zip(names, demangle(names), blocks):
            if not any(re.search(re.escape(p) if '<' in p and '\\' not in p else p, dem) for p in pats):
                continue
            ins = re.findall(r'/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)', blk)

            def cnt(rx):
                return sum(1 for i in ins if re.match(rx, i))
            reg, stack, shared, local = usage.get(name, (None, None, None, None))
            rows.append((dem, len(ins), cnt(r'UBLKCP'), cnt(r'LDG\.E.*\.128'), cnt(r'STG\.E.*\.128'), cnt(r'LDG'), cnt(r'STG'),
                         cnt(r'IMAD\.WIDE'), cnt(r'IMAD'), cnt(r'IADD3|IADD'), cnt(r'LOP3|SHF|SEL'), cnt(r'LDS|STS'), cnt(r'LDGSTS'),
                         cnt(r'HMMA|IMMA|UTCMMA|UTMALDG'), reg, stack, local, shared))
    hdr = ('kernel', 'SASS', 'UBLKCP', 'LDG128', 'STG128', 'LDG', 'STG', 'IMAD.W', 'IMAD*', 'IADD3', 'LOP/SHF/SEL', 'LDS/STS', 'LDGSTS', 'tensor', 'regs',
           'stack', 'local', 'smem')
    print('# static SASS / resource summary of the hot kernels (sm_90a), tools/sass_summary.py')
    print(('%-44s' + ' %7s' * (len(hdr) - 1)) % hdr)
    for r in sorted(rows):
        print(('%-44s' + ' %7s' * (len(r) - 1)) % r)


if __name__ == '__main__':
    main()
