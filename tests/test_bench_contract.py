"""The JSON-line contract of bench.py that can be checked without a GPU: the reference arm (`--impl reference`: the
unmodified reference where it is importable -- oracle/_ref or $MPYC_REFERENCE --, else the oracle port) prints one line
with the keys the driver reads, on the same `config` as the GPU arm, with an `e2e` that moves no bytes over PCIe."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_the_contract_line():
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'bench.py'), '--impl', 'reference', '--steps', '1', '--warmup', '1'],
                       capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    for key in ('metric', 'value', 'unit', 'n_gpus', 'steps', 'warmup', 'ms_per_step', 'higher_is_better', 'scaling', 'vs_baseline',
                'dtype', 'data', 'config', 'cpu_baseline', 'e2e', 'impl'):
        assert key in line, key
    assert line['impl'] == 'reference' and line['unit'] == 'pairs/s' and line['higher_is_better'] is True
    assert line['value'] > 0 and line['steps'] == 1 and line['n_gpus'] == 1 and line['vs_baseline'] is None
    cfg = line['config']
    assert 'workload' in cfg and cfg['p_bits'] == 128 and cfg['m'] == 5 and cfg['t'] == 2 and cfg['recombine_k'] == 3
    cb = line['cpu_baseline']
    assert cb['kind'] in ('reference', 'port') and cb['cores'] >= 1 and cb['value'] == line['value'] and cb['sample']
    e2e = line['e2e']
    assert e2e['value'] == line['value'] and e2e['h2d_bytes_per_step'] == 0 and e2e['d2h_bytes_per_step'] == 0


def test_dump_outputs_samples_fixed_indices_as_exact_words(tmp_path, monkeypatch):
    """--dump-outputs: one ascending element sample for every array and run, 64-bit limbs as exact 32-bit words in
    float64, GF(2^8) bytes as values; the largest workload (7 shares + 1 recombined row of 4 limbs) stays under 64 MB."""
    import numpy as np
    import torch
    sys.path.insert(0, ROOT)
    import bench
    n, k = 1000, -0x100000003
    limbs = (torch.arange(1, n + 1) * k)[None, :, None] * torch.tensor([1, 2, 3])[:, None, None].repeat(1, 1, 2)
    gf = (torch.arange(n) % 251).to(torch.uint8)[None]
    assert 8 * bench.DUMP_SAMPLE * 4 * 2 * 8 <= 64 << 20
    for run, sample in (('a', bench.DUMP_SAMPLE), ('b', bench.DUMP_SAMPLE), ('c', 64)):
        monkeypatch.setattr(bench, 'DUMP_SAMPLE', sample)
        bench.dump_outputs(str(tmp_path / run), {'shares': limbs, 'recombined': limbs[1], 'bytes': gf}, n)
    a, b, c = ({f: np.load(tmp_path / r / f'{f}.npy') for f in ('shares', 'recombined', 'bytes')} for r in 'abc')
    assert all(a[f].dtype == np.float64 and (a[f] == b[f]).all() for f in a)
    assert (a['shares'] == limbs.numpy().view(np.uint32)).all() and (a['bytes'] == gf.numpy()).all()
    w = c['shares'][0].astype(np.uint64)
    picked = (w[:, 0] + (w[:, 1] << 32)).view(np.int64) // k
    assert c['shares'].shape == (3, 64, 4) and (np.diff(picked) > 0).all() and (c['recombined'] == c['shares'][1]).all()
