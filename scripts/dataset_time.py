#!/usr/bin/env python3
"""Times pb_score_dataset (labelled clips, DESIGN.md section 6) against the loop it replaces.

    python scripts/dataset_time.py [--clips 100000] [--seconds 3] [--models 1,64,1024] [--loop-models 8] [--rounds 3]

Clips are views of one seeded noise buffer on the device, all of one length; a third of them are labelled wake word.  k pool
models cycle over 64 seeded default-shaped networks.  Arms, per k:
  loop   for each of min(k, --loop-models) models: offline.vectorize of every clip (batches of 2 048 clips through pb_mfcc)
         and one pb_predict over all of them, outputs copied to the host; reported per model
  stats  pb_score_dataset without d_raw: counts, a 98-threshold histogram (precise-graph's) and the fit sums; only the
         statistics are copied to the host
  raw    the same with d_raw [k, clips], and raw copied to the host as well
Clips are packed once, outside the timed region (offline._pack_clips, calls of at most offline.CORPUS_CALL_SAMPLES samples).
Times are host clocks around work that ends in a device synchronise, lowest - highest of the rounds after a warm-up.
Prints the card, its power limit and one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--clips', type=int, default=100000)
    ap.add_argument('--seconds', type=float, default=3.0)
    ap.add_argument('--models', default='1,64,1024')
    ap.add_argument('--loop-models', type=int, default=8)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    import torch
    import mycroft_precise_b200 as m
    from mycroft_precise_b200 import offline
    assert torch.cuda.is_available(), 'needs a GPU'
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                          capture_output=True, text=True).stdout.strip()
    print('card:', card)
    ks = [int(v) for v in args.models.split(',')]
    nets = [m.GruModel.random(13, 20, seed=i, scale=0.1) for i in range(64)]
    core = m.PreciseB200()
    core.set_pool(64)
    for i, g in enumerate(nets):
        core.pool_load(i, g)
    loop = m.PreciseB200()
    L = int(args.seconds * 16000)
    gen = torch.Generator(device='cuda').manual_seed(0)
    buf = (torch.randn(1 << 27, device='cuda', generator=gen) * 3000).clamp_(-32768, 32767).to(torch.int16)
    starts = np.random.RandomState(0).randint(0, buf.numel() - L, args.clips)
    clips = [buf[s:s + L] for s in starts.tolist()]
    targets = (np.arange(args.clips) % 3 == 0).astype(np.uint8)
    thr = offline.graph_thresholds(core.params).astype(np.float64)
    calls = []
    first = 0
    for g in offline._call_groups([c[-core.params.max_samples:] for c in clips]):
        pcm, offsets, order = offline._pack_clips(core, g)
        calls.append((pcm, offsets, np.ascontiguousarray(targets[first + order])))
        first += len(g)
    sync = torch.cuda.synchronize

    def arm_dataset(ids, per_entry):
        out = []
        for pcm, offsets, tg in calls:
            res = core.score_dataset(pcm, offsets, tg, ids, thresholds=thr, per_entry=per_entry)
            out.append([res[key].cpu() for key in ('count', 'hist', 'fit') + (('raw',) if per_entry else ())])
        sync()
        return out

    def arm_loop(n_models):
        for i in range(n_models):
            g = nets[i % 64]
            loop.load_weights(g.kernel, g.recurrent, g.bias, g.dense_w, g.dense_b)
            feats = [offline.vectorize(loop, torch.stack(clips[a:a + 2048])) for a in range(0, len(clips), 2048)]
            loop.predict(torch.cat(feats)).cpu()
        sync()

    def timed(fn):
        fn()
        ts = []
        for _ in range(args.rounds):
            sync()
            t0 = time.perf_counter()
            fn()
            ts.append((time.perf_counter() - t0) * 1e3)
        return min(ts), max(ts)

    rows = []
    for k in ks:
        ids = (np.arange(k) % 64).astype(np.int32)
        nl = min(k, args.loop_models)
        lo = timed(lambda: arm_loop(nl))
        st = timed(lambda: arm_dataset(ids, False))
        rw = timed(lambda: arm_dataset(ids, True))
        core.profile(True)
        arm_dataset(ids, False)
        prof_ms, _ = core.profile_read()
        core.profile(False)
        rows.append(dict(k=k, clips=args.clips, seconds=args.seconds, calls=len(calls), loop_models=nl,
                         loop_ms_per_model=[v / nl for v in lo], stats_ms=st, raw_ms=rw, k1_ms=prof_ms[0], scan_stats_ms=prof_ms[1],
                         stats_entries_per_s=k * args.clips / (st[1] / 1e3)))
        print('k = %5d: loop %.1f-%.1f ms per model (%d models), stats %.1f-%.1f ms, raw + readback %.1f-%.1f ms, K1 %.2f ms, '
              'scans + statistics %.2f ms' % (k, lo[0] / nl, lo[1] / nl, nl, st[0], st[1], rw[0], rw[1], prof_ms[0], prof_ms[1]))
    print(json.dumps(dict(card=card, rows=rows)))
    core.close()
    loop.close()


if __name__ == '__main__':
    main()
