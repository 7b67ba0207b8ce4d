"""In-tree build of libmpyc_b200.so (sm_90a) with nvcc.  No torch involved: the library is plain CUDA
behind a C ABI.  Objects go to mpyc_b200/csrc/_obj/, the shared library next to this file."""
import concurrent.futures
import hashlib
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OBJ = os.path.join(CSRC, '_obj')
LIB = os.path.join(HERE, 'libmpyc_b200.so')
SOURCES = ['api.cu', 'inst_L1.cu', 'inst_L2.cu', 'inst_L3.cu', 'inst_L4.cu', 'inst_layout.cu', 'inst_linalg.cu', 'inst_conv.cu',
           'inst_select.cu', 'inst_powexp.cu', 'inst_prod.cu', 'inst_matmul_int.cu', 'inst_gf.cu']
HOST_SOURCES = ['shake128_x8.cpp']   # host compiler only (AVX-512 through per-function target attributes)
PUBLIC_HEADER = os.path.join('..', '..', 'include', 'mpyc_b200.h')


def _headers():
    """Every header a translation unit may include: all of csrc/*.h, *.cuh plus the public C header."""
    return sorted(f for f in os.listdir(CSRC) if f.endswith(('.h', '.cuh'))) + [PUBLIC_HEADER]
NVCC_FLAGS = ['-std=c++17', '-O3', '-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo',
              '-Xcompiler', '-fPIC', '-Xcompiler', '-fvisibility=hidden', '-Xcompiler', '-fno-strict-aliasing', '--expt-relaxed-constexpr',
              '-Xfatbin', '-compress-all']   # compressed fatbin: a smaller library to load and ship


def _nvcc():
    cand = shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'
    if not os.path.exists(cand):
        raise RuntimeError('nvcc not found: cannot build libmpyc_b200.so')
    return cand


def _digest():
    h = hashlib.sha256(' '.join(NVCC_FLAGS).encode())
    for name in SOURCES + HOST_SOURCES + _headers():
        with open(os.path.join(CSRC, name), 'rb') as fh:
            h.update(fh.read())
    return h.hexdigest()


CODEC_SRC = os.path.join(CSRC, 'pycodec.c')
CODEC_LIB = os.path.join(HERE, '_pycodec.so')


def _codec_digest():
    """Source hash + the interpreter's ABI: pycodec.c reads CPython's long-object digits directly, so an extension
    built for another interpreter must never be loaded (it is rebuilt instead)."""
    import sys
    import sysconfig
    h = hashlib.sha256()
    with open(CODEC_SRC, 'rb') as fh:
        h.update(fh.read())
    h.update(repr((sys.implementation.name, sys.version_info[:3], sysconfig.get_config_var('EXT_SUFFIX'),
                   sys.int_info.bits_per_digit)).encode())
    return h.hexdigest()


def build_codec(force=False):
    """The small CPython extension that packs/unpacks Python ints (gcc, no CUDA involved)."""
    import sysconfig
    stamp = CODEC_LIB + '.digest'
    digest = _codec_digest()
    if not force and os.path.exists(CODEC_LIB) and os.path.exists(stamp) and open(stamp).read() == digest:
        return CODEC_LIB
    inc = sysconfig.get_paths()['include']
    r = subprocess.run(['gcc', '-O2', '-shared', '-fPIC', '-I' + inc, CODEC_SRC, '-o', CODEC_LIB], capture_output=True, text=True)
    if r.returncode:
        raise RuntimeError('gcc failed for pycodec.c:\n' + r.stderr[-4000:])
    with open(stamp, 'w') as fh:
        fh.write(digest)
    return CODEC_LIB


def build(force=False, verbose=False, defines=(), lib=None):
    """Compile (if sources changed) and return the path of the shared library.
    defines/lib: build a tuning variant (-D flags) under another file name (kernel experiments)."""
    global OBJ, LIB
    if lib is not None:
        saved = (OBJ, LIB)
        OBJ, LIB = os.path.join(CSRC, '_obj_' + os.path.basename(lib)), os.path.join(HERE, lib)
        try:
            return build(force=True, verbose=verbose, defines=defines)
        finally:
            OBJ, LIB = saved
    os.makedirs(OBJ, exist_ok=True)
    stamp = LIB + '.digest'   # next to the library, so that the pair can be moved together
    digest = _digest()

    def fresh():
        return os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == digest
    if not force and fresh():
        build_codec(force=False)
        return LIB
    # several processes may import the package at once (torchrun ranks, MPyC parties): one of them builds, the others wait
    # on the lock and then find the fresh stamp
    import fcntl
    with open(os.path.join(OBJ, '.build.lock'), 'w') as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            build_codec(force=False)
            if not force and fresh():
                return LIB
            return _build_locked(verbose, defines, stamp, digest)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)


def _build_locked(verbose, defines, stamp, digest):
    nvcc = _nvcc()

    def compile_one(src):
        obj = os.path.join(OBJ, src.replace('.cu', '.o'))
        cmd = [nvcc] + NVCC_FLAGS + ['-D' + d for d in defines] + (['-Xptxas', '-v'] if verbose else []) + ['-c', os.path.join(CSRC, src), '-o', obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode:
            raise RuntimeError('nvcc failed for %s:\n%s\n%s' % (src, r.stdout[-4000:], r.stderr[-8000:]))
        return obj, r.stderr

    def compile_host(src):
        obj = os.path.join(OBJ, src.replace('.cpp', '.o'))
        r = subprocess.run(['g++', '-std=c++17', '-O3', '-fPIC', '-fvisibility=hidden', '-c', os.path.join(CSRC, src), '-o', obj],
                           capture_output=True, text=True)
        if r.returncode:
            raise RuntimeError('g++ failed for %s:\n%s' % (src, r.stderr[-4000:]))
        return obj, r.stderr

    with concurrent.futures.ThreadPoolExecutor(max_workers=len(SOURCES) + len(HOST_SOURCES)) as ex:
        host_jobs = [ex.submit(compile_host, src) for src in HOST_SOURCES]
        results = list(ex.map(compile_one, SOURCES)) + [j.result() for j in host_jobs]
    objs = [o for o, _ in results]
    if verbose:
        with open(os.path.join(OBJ, 'ptxas.log'), 'w') as fh:
            for _, err in results:
                fh.write(err)
    r = subprocess.run([nvcc, '-shared', '-o', LIB] + objs + ['-lcudart_static', '-ldl', '-lrt', '-lpthread'],
                       capture_output=True, text=True)
    if r.returncode:
        raise RuntimeError('link failed:\n' + r.stderr[-4000:])
    with open(stamp, 'w') as fh:
        fh.write(digest)
    return LIB


if __name__ == '__main__':
    import sys
    defs = [a[2:] for a in sys.argv[1:] if a.startswith('-D')]
    out = [a[2:] for a in sys.argv[1:] if a.startswith('-o')]
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv, defines=defs, lib=out[0] if out else None))
