"""Memory ceilings of K2's and K3's read/write mixes on this card (tools/stream_probe.cu, no arithmetic).

Builds the probe with nvcc into a temporary directory, runs it, and prints the card's name and power limit with one
line per mix and access form (GB/s counts every row read and written) and a 2 GiB device copy.

    python tools/stream_probe.py [--reps 20] [--json OUT]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))


def card():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=60)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--reps', type=int, default=20, help='timed launches per measurement (after 3 warm-up launches)')
    ap.add_argument('--json', metavar='OUT', help='also write the records (and the card) to this file')
    a = ap.parse_args()
    nvcc = shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, 'stream_probe')
        subprocess.run([nvcc, '-O3', '-std=c++17', '-gencode', 'arch=compute_90a,code=sm_90a',
                        os.path.join(HERE, 'stream_probe.cu'), '-o', exe], check=True)
        out = subprocess.run([exe, str(a.reps)], capture_output=True, text=True, check=True).stdout
    recs = [json.loads(line) for line in out.splitlines() if line.startswith('{')]
    name = card()
    print(f'card: {name}')
    print(f'{"mix":10} {"in/out":>6} {"form":>10} {"ms":>8} {"GB/s":>7}')
    for r in recs:
        print(f'{r["mix"]:10} {r["in"]:>3}/{r["out"]:<2} {r["form"]:>10} {r["ms"]:8.3f} {r["GBps"]:7.0f}')
    if a.json:
        with open(a.json, 'w') as fh:
            json.dump({'card': name, 'records': recs}, fh, indent=1)
    return 0


if __name__ == '__main__':
    sys.exit(main())
