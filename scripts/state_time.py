"""Stream state export / import at the bench size (DESIGN.md §3 "Stream state export / import", §6).

131 072 streams of the default geometry, a default-shaped network (H = 20 over 13 MFCCs) with seeded weights, seeded PCM,
primed with PRIME ticks.  Each round exports every stream in a permuted id order (pb_export_streams, asynchronous: CUDA events
around ITERS exports) and imports the records into a second handle at the same ids (pb_import_streams, synchronous: CUDA
events around each call, which includes the validation kernel and its read-back).  Rounds alternate export and import.  The
byte model is n x record bytes read plus n x record bytes written per call (import's validation also reads 64 B per record).
After the rounds both handles take the same tick: raw, conf, fired and the counts must be bit-identical.

    python scripts/state_time.py [--out result.json]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np                      # noqa: E402
import torch                            # noqa: E402
import mycroft_precise_b200 as m        # noqa: E402
from bank_time import S, PRIME, card    # noqa: E402

ITERS, REPS = 10, 4


def same_bits(x, y):
    x, y = x.contiguous(), y.contiguous()
    return x.shape == y.shape and bool(torch.equal(x.view(torch.uint8), y.view(torch.uint8)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='also write the results as JSON to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('state_time.py needs a CUDA device')
    gpu = card()
    print('card:', gpu, flush=True)
    model = m.GruModel.random(13, 20, seed=0, scale=0.1)
    model.dense_b = 3.0                     # streams fire, so activations are non-zero
    pcm = [torch.from_numpy(np.clip(np.random.RandomState(i).randn(S, 1024) * 3000, -32768, 32767).astype(np.int16)).cuda()
           for i in range(3)]
    a, b = m.StreamBatch(model, S), m.StreamBatch(model, S)
    for i in range(PRIME):
        a.update(pcm[i & 1])
    perm = np.random.RandomState(7).permutation(S).astype(np.int32)
    ids = torch.from_numpy(perm).cuda()
    R = a.core.stream_state_bytes
    out = torch.empty((S, R), dtype=torch.uint8, device='cuda')
    a.core.export_streams(ids, out=out)                 # warm-up of both kernels
    b.core.import_streams(out, perm)
    torch.cuda.synchronize()
    moved = 2.0 * S * R                                 # bytes read + written per call
    results = []
    for rep in range(REPS):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(ITERS):
            a.core.export_streams(ids, out=out)
        t1.record()
        torch.cuda.synchronize()
        exp_us = t0.elapsed_time(t1) * 1e3 / ITERS
        imp = []
        for _ in range(ITERS):
            t0.record()
            b.core.import_streams(out, perm)
            t1.record()
            torch.cuda.synchronize()
            imp.append(t0.elapsed_time(t1) * 1e3)
        imp_us = float(np.median(imp))
        row = dict(round=rep, export_us=exp_us, export_gbs=moved / exp_us * 1e-3, import_us=imp_us,
                   import_gbs=moved / imp_us * 1e-3, import_us_min=float(min(imp)))
        print('round %d  export %7.1f us  %6.0f GB/s   import (whole call) %7.1f us (min %7.1f)  %6.0f GB/s'
              % (rep, exp_us, row['export_gbs'], imp_us, row['import_us_min'], row['import_gbs']), flush=True)
        results.append(row)
    oa, ob = a.update(pcm[2]), b.update(pcm[2])
    ok = all(same_bits(oa[k], ob[k]) for k in ('raw', 'conf', 'fired'))
    a.reset_count()
    b.reset_count()
    oa, ob = a.update(pcm[0]), b.update(pcm[0])
    ok = ok and all(same_bits(oa[k], ob[k]) for k in ('raw', 'conf', 'fired')) and same_bits(a.count, b.count)
    print('record %d B, %d streams, %.1f MB per direction; next ticks bit-identical: %s (count %d)'
          % (R, S, S * R / 1e6, ok, int(a.count.item())), flush=True)
    assert ok
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(dict(card=gpu, streams=S, record_bytes=R, prime=PRIME, iters=ITERS, results=results), f, indent=1)
    for x in (a, b):
        x.core.close()


if __name__ == '__main__':
    main()
