"""K2 of the default tick, one library build against another (DESIGN.md §3 "K2+K3", §6).

131 072 streams, the default network (H = 20 over 13 MFCCs) with seeded weights, seeded PCM, one `update` per tick.  Each arm is
a build of libprecise_b200.so, loaded through PRECISE_B200_LIB in a subprocess of its own; the arms alternate, ROUNDS rounds
each.  A round primes PRIME untimed ticks (full 29-frame windows from tick 24 on), then times TIMED ticks: K1 / K2 from the
library's CUDA-event profile (pb_profile_*, slots 0 / 1), the tick from CUDA events around the timed loop.  Every round sees the
same tick sequence, so the last tick's raw / conf / fired must be bit-identical across all arms and rounds.

K2's floors come from what the scan has to do per update (bench.py's roofline_k2 block models an older kernel):
  bytes  K2_BYTES_PER_UPDATE = 29 ring rows x 64 B + raw (4) + conf (8) + fired (1) + trigger state (4 read + 4 written)
  FLOP   K2_MMA_FLOP_PER_UPDATE = 9 n-tiles x 3 passes x 29 steps x (m16n8k16 for x.W + m16n8k16 and m16n8k8 for h.U) / 16 streams
         K2_WGMMA_FLOP_PER_UPDATE: the same with the k8 products run as k16 (what gru_wg_kernel executes)
against the H100 SXM data sheet (3.35 TB/s HBM3, 989 TFLOP/s dense fp16).

The parent commit's library, for the default comparison:
    mkdir -p build/parent && git archive <parent> mycroft_precise_b200/csrc include | tar -x -C build/parent
    make -C build/parent/mycroft_precise_b200/csrc
    python scripts/k2_time.py [--arm NAME=LIB ...] [--rounds 3] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
S, PRIME, TIMED = 131072, 30, 50
K2_BYTES_PER_UPDATE = 29 * 64 + 4 + 8 + 1 + 4 + 4                      # 1 877
K2_MMA_FLOP_PER_UPDATE = 9 * 3 * 29 * (2 * 16 * 8 * 16 + 2 * 16 * 8 * 16 + 2 * 16 * 8 * 8) // 16   # 501 120
K2_WGMMA_FLOP_PER_UPDATE = 9 * 3 * 29 * (3 * 2 * 16 * 8 * 16) // 16                         # 601 344: k8 groups run as k16 on wgmma
HBM_BPS, FP16_FLOPS = 3.35e12, 989e12
DEFAULT_ARMS = ['parent=' + os.path.join(ROOT, 'build', 'parent', 'mycroft_precise_b200', 'csrc', 'libprecise_b200.so'),
                'tree=' + os.path.join(ROOT, 'mycroft_precise_b200', 'csrc', 'libprecise_b200.so')]


def card():
    """Name, power limit and max SM clock of cuda:0, read in the same run as the timings."""
    try:
        q = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ''
    return q or 'power limit not readable'


def child(dump):
    """One round on the library PRECISE_B200_LIB names: prints one JSON line, writes the last tick's outputs under dump."""
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    import mycroft_precise_b200 as m
    if not torch.cuda.is_available():
        sys.exit('k2_time.py needs a CUDA device')
    sb = m.StreamBatch(m.GruModel.random(13, 20, seed=0, scale=0.1), S)
    pcm = [torch.from_numpy(np.clip(np.random.RandomState(i).randn(S, 1024) * 3000, -32768, 32767).astype(np.int16)).cuda()
           for i in range(2)]
    for i in range(PRIME):
        sb.update(pcm[i & 1])
    torch.cuda.synchronize()
    sb.core.profile(True)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for i in range(TIMED):
        out = sb.update(pcm[(PRIME + i) & 1])
    t1.record()
    torch.cuda.synchronize()
    ms, launches = sb.core.profile_read()
    for k in ('raw', 'conf', 'fired'):
        np.save(os.path.join(dump, k + '.npy'), out[k].cpu().numpy())
    us = 1e3 / TIMED
    print(json.dumps(dict(k1_us=ms[0] * us, k2_us=ms[1] * us, tick_us=t0.elapsed_time(t1) * us, k2_launches=launches[1],
                          lib=sb.core.lib.pb_build_info().decode(), gpu=torch.cuda.get_device_name(0))), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--arm', action='append', default=None, help='NAME=path of a libprecise_b200.so (repeatable)')
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None, help='also write the results as JSON to this file')
    ap.add_argument('--child', default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args.child)
    arms = [a.split('=', 1) for a in (args.arm or DEFAULT_ARMS)]
    for name, lib in arms:
        if not os.path.isfile(lib):
            sys.exit('arm %s: %s is missing' % (name, lib))
    gpu = card()
    print('card (name, power limit, max SM clock):', gpu, flush=True)
    import numpy as np
    results, ref = [], None
    for rnd in range(args.rounds):
        for name, lib in arms:
            with tempfile.TemporaryDirectory() as dump:
                p = subprocess.run([sys.executable, os.path.abspath(__file__), '--child', dump],
                                   env=dict(os.environ, PRECISE_B200_LIB=os.path.abspath(lib)), capture_output=True, text=True)
                if p.returncode != 0:
                    sys.exit('arm %s round %d failed:\n%s%s' % (name, rnd, p.stdout, p.stderr))
                r = json.loads(p.stdout.strip().splitlines()[-1])
                outs = {k: np.load(os.path.join(dump, k + '.npy')) for k in ('raw', 'conf', 'fired')}
            if ref is None:
                ref = outs
            same = all(np.array_equal(outs[k].view(np.uint8), ref[k].view(np.uint8)) for k in outs)
            sec = r['k2_us'] * 1e-6
            r.update(arm=name, round=rnd, outputs_match_first=same,
                     k2_GBps=S * K2_BYTES_PER_UPDATE / sec / 1e9, k2_TFLOPs=S * K2_MMA_FLOP_PER_UPDATE / sec / 1e12,
                     k2_wgmma_TFLOPs=S * K2_WGMMA_FLOP_PER_UPDATE / sec / 1e12)
            r['k2_frac_of_floor'] = max(S * K2_BYTES_PER_UPDATE / HBM_BPS, S * K2_MMA_FLOP_PER_UPDATE / FP16_FLOPS) / sec
            print('round %d %-8s K1 %6.1f us  K2 %6.1f us  tick %6.1f us | K2 %5.0f GB/s  %5.1f TFLOP/s  %.0f %% of the floor | '
                  'outputs bit-identical to the first run: %s'
                  % (rnd, name, r['k1_us'], r['k2_us'], r['tick_us'], r['k2_GBps'], r['k2_TFLOPs'], 100 * r['k2_frac_of_floor'], same),
                  flush=True)
            results.append(r)
    for name, _ in arms:
        k2 = [r['k2_us'] for r in results if r['arm'] == name]
        tick = [r['tick_us'] for r in results if r['arm'] == name]
        print('%-8s K2 %.1f .. %.1f us   tick %.1f .. %.1f us' % (name, min(k2), max(k2), min(tick), max(tick)))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(dict(card=gpu, streams=S, prime=PRIME, timed=TIMED, bytes_per_update=K2_BYTES_PER_UPDATE,
                           mma_flop_per_update=K2_MMA_FLOP_PER_UPDATE,
                           wgmma_flop_per_update=K2_WGMMA_FLOP_PER_UPDATE, results=results), f, indent=1)
    if not all(r['outputs_match_first'] for r in results):
        sys.exit('outputs differ between runs')


if __name__ == '__main__':
    main()
