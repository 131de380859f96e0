"""Times pb_score_rows (csrc/rows.cuh) against the loop it replaces, and against the pool path for fused networks.

    python scripts/rows_time.py [--out FILE.json] [--quick]

1. Rows against the loop: k in {1, 8, 64, 256} networks of H in {24, 64, 128} units over n in {2 000, 20 000} network
   inputs at the default front end (F = 13, T = 29), thresholds (0.5,), count, hist, fit and misses.  The loop is what a
   user wrote before: per network pb_load_weights (the host-side TF32 split and upload) and pb_predict, then the same
   statistics on the device in torch (counts per label, #(raw > 0.5) per label, calc_threshold's fit sums, the mask and
   number of misclassified entries) from masked sums only, so that nothing but pb_load_weights' uploads waits between
   networks.
2. Rows against the pool for fused networks (H 20): pb_score_dataset over the clips' PCM (its own MFCC pass) against
   pb_vectorize_clips + pb_score_rows, k in {1, 8, 64, 256}, 2 000 and 20 000 one-second noise clips.

Inputs are seeded noise; the scan's cost does not depend on their values.  Times are CUDA events around one call after a
warm-up call of the same shape, the best of three.  The miss lists have room for every entry, so no call runs twice.  The card's name, power limit and maximum SM clock are read in the same
run.  --quick: k = 1 and 64, n = 2 000 only.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

T, F = 29, 13


def timed(torch, fn, reps=3):
    fn()                                                          # warm-up
    torch.cuda.synchronize()
    best = float('inf')
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        best = min(best, a.elapsed_time(b) / 1e3)
    return best


def torch_stats(torch, raw, y):
    """The loop's statistics of one network on the device: what pb_score_rows returns for thresholds (0.5,)."""
    pos = y != 0
    above = raw > 0.5
    t = 1.0 / raw - 1.0
    ok = (raw != 0) & (raw != 1) & torch.isfinite(t.log())
    v = -t.double().log()
    v = torch.where(ok & pos, v, torch.zeros_like(v))
    miss = above != pos
    return (pos.sum(), (~pos).sum(), (above & pos).sum(), (above & ~pos).sum(), (ok & pos).sum(), v.sum(), (v * v).sum(),
            miss, miss.sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out')
    ap.add_argument('--quick', action='store_true')
    args = ap.parse_args()
    import torch
    import mycroft_precise_b200 as m
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print('card:', card)
    ks = (1, 64) if args.quick else (1, 8, 64, 256)
    ns = (2000,) if args.quick else (2000, 20000)
    core = m.PreciseB200()
    out = dict(card=card, rows=[], pool=[])
    gen = torch.Generator('cuda').manual_seed(0)
    for n in ns:
        x = torch.randn((n, T, F), device='cuda', generator=gen) * 5
        y = (np.arange(n) % 4 == 0).astype(np.uint8)
        yd = torch.from_numpy(y).cuda()
        for H in (24, 64, 128):
            handle = m.PreciseB200(hidden=H, activation='linear', recurrent_activation='hard_sigmoid')
            for k in ks:
                models = [m.GruModel.random(F, H, seed=i, scale=0.1) for i in range(k)]
                st = m.offline.TrainState.from_models(core, models, list(range(k)))
                t_rows = timed(torch, lambda: core.score_rows(x, y, st.rows, st.weights, per_entry=False, miss_threshold=0.5,
                                                              miss_capacity=k * n))

                def loop():
                    for g in models:
                        handle.load_weights(g.kernel, g.recurrent, g.bias, g.dense_w, g.dense_b)
                        torch_stats(torch, handle.predict(x).view(-1), yd)
                t_loop = timed(torch, loop)
                r = dict(n=n, H=H, k=k, rows_s=t_rows, loop_s=t_loop, speedup=t_loop / t_rows,
                         entries_per_s=k * n / t_rows)
                out['rows'].append(r)
                print('rows  n %6d  H %3d  k %3d   rows %8.4f s   loop %8.4f s   x%.2f   %.3g entries/s'
                      % (n, H, k, t_rows, t_loop, r['speedup'], r['entries_per_s']), flush=True)
            handle.close()
        # fused networks: the pool path from PCM against vectorize + rows
        L = 16000
        pcm = (torch.randn(n * L, device='cuda', generator=gen) * 3000).clamp(-32768, 32767).to(torch.int16)
        offsets = np.arange(n + 1, dtype=np.int64) * L
        for k in ks:
            models = [m.GruModel.random(F, 20, seed=i, scale=0.1) for i in range(k)]
            core.set_pool(k)
            for i, g in enumerate(models):
                core.pool_load(i, g)
            ids = np.arange(k, dtype=np.int32)
            st = m.offline.TrainState.from_models(core, models, list(range(k)))
            t_pool = timed(torch, lambda: core.score_dataset(pcm, offsets, y, ids, per_entry=False, miss_threshold=0.5,
                                                             miss_capacity=k * n))
            t_vr = timed(torch, lambda: core.score_rows(core.vectorize_clips(pcm, offsets), y, st.rows, st.weights,
                                                        per_entry=False, miss_threshold=0.5, miss_capacity=k * n))
            xv = core.vectorize_clips(pcm, offsets)
            t_r = timed(torch, lambda: core.score_rows(xv, y, st.rows, st.weights, per_entry=False, miss_threshold=0.5,
                                                       miss_capacity=k * n))
            r = dict(n=n, H=20, k=k, pool_s=t_pool, vectorize_rows_s=t_vr, rows_s=t_r)
            out['pool'].append(r)
            print('pool  n %6d  H  20  k %3d   pool %8.4f s   vectorize+rows %8.4f s   rows alone %8.4f s'
                  % (n, k, t_pool, t_vr, t_r), flush=True)
        del pcm
    core.close()
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
