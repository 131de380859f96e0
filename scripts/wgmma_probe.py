"""Builds and runs scripts/wgmma_probe.cu (DESIGN.md §6 "wgmma probe"): the default scan's per-step products on mma.sync and
on wgmma, their rate and latency on one SM, and their bit equality.  Prints one JSON line with the card's name, power limit
and clocks read in the same run.

    python scripts/wgmma_probe.py [--steps 4096] [--eq-iters 24] [--out probe.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    q = ['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader']
    try:
        out = subprocess.run(q, capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ''
    return out or 'not readable'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=4096)
    ap.add_argument('--eq-iters', type=int, default=24, help='equality iterations per CTA (64 x 24 cases each)')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    nvcc = os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'nvcc')
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, 'wgmma_probe')
        subprocess.run([nvcc, '-O3', '-std=c++17', '-gencode', 'arch=compute_90a,code=sm_90a', '-o', exe,
                        os.path.join(ROOT, 'scripts', 'wgmma_probe.cu')], check=True)
        before = card()
        p = subprocess.run([exe, str(args.steps), str(args.eq_iters)], capture_output=True, text=True)
        after = card()
    if p.returncode != 0:
        sys.exit('wgmma_probe failed:\n' + p.stdout + p.stderr)
    r = json.loads(p.stdout.strip().splitlines()[-1])
    r['nvidia_smi_before'] = before                    # name, power limit, SM clock, max SM clock
    r['nvidia_smi_after'] = after
    r['go'] = r['wgmma_over_mma_sync'] >= 1.6 and r['eq_mismatches'] == 0 and r['scan_h_bit_differences'] == 0
    line = json.dumps(r)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
