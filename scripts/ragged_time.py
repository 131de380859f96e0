"""Ragged ticks at the bench size (DESIGN.md §3 "Ragged ticks", §6).

131 072 streams, the default network (H = 20 over 13 MFCCs) with seeded weights and seeded PCM.
  arm a: update, uniform 1024-sample chunks;
  arm b: update_ragged with every length 1024 on a fresh handle (aligned offsets, the ragged MFCC kernel);
  arm c: update_ragged with lengths drawn from [768, 1280] (mean 1024) after one odd filler sample, so offsets are odd;
  arm d: arm c with force_generic (the generic MFCC kernel).
The arms alternate in one process (REPS rounds).  Each round primes PRIME untimed ticks, then times TIMED ticks: K1 / K2 from the
library's CUDA-event profile (pb_profile_*, slots 0 / 1), tick time from CUDA events around the timed loop.  Arms a and b see the
same ticks and must dump bit-identical raw, conf and fired; arms c and d must agree within 1e-5 on raw.

    python scripts/ragged_time.py [--out result.json]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np                      # noqa: E402
import torch                            # noqa: E402
import mycroft_precise_b200 as m        # noqa: E402
from bank_time import card, timed       # noqa: E402  (scripts/ is on sys.path when this file runs)

S, REPS = 131072, 2


def ragged_input(seed):
    rs = np.random.RandomState(seed)
    lens = rs.randint(768, 1281, size=S).astype(np.int64)
    offs = 1 + np.concatenate([[0], np.cumsum(lens)])
    pcm = np.clip(rs.randn(int(offs[-1])) * 3000, -32768, 32767).astype(np.int16)
    return torch.from_numpy(pcm).cuda(), torch.from_numpy(offs).cuda(), int(lens.max())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='also write the results as JSON to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('ragged_time.py needs a CUDA device')
    gpu = card()
    print('card:', gpu, flush=True)
    model = m.GruModel.random(13, 20, seed=0, scale=0.1)
    pcm = [torch.from_numpy(np.clip(np.random.RandomState(i).randn(S, 1024) * 3000, -32768, 32767).astype(np.int16)).cuda()
           for i in range(2)]
    aligned = torch.arange(S + 1, dtype=torch.int64, device='cuda') * 1024
    rag = [ragged_input(10 + i) for i in range(2)]
    a, b, c, d = (m.StreamBatch(model, S) for _ in range(4))
    d.core.force_generic(True)
    arms = dict(a=(a, lambda p: a.update(p)),
                b=(b, lambda p: b.update_ragged(p.view(-1), aligned, max_len=1024)),
                c=(c, lambda r: c.update_ragged(r[0], r[1], max_len=r[2])),
                d=(d, lambda r: d.update_ragged(r[0], r[1], max_len=r[2])))
    results = []
    for rep in range(REPS):
        row = {}
        outs = {}
        for name, (sb, tick) in arms.items():
            t, o = timed([sb], tick, pcm if name in 'ab' else rag)
            row[name] = t
            outs[name] = {k: v.clone() for k, v in o.items()}
        same_ab = all(torch.equal(outs['a'][k], outs['b'][k].view(-1)) for k in ('raw', 'conf', 'fired'))
        err_cd = float((outs['c']['raw'] - outs['d']['raw']).abs().max())
        print('round %d  ' % rep + '  '.join('%s: K1 %.1f us  K2 %.1f us  tick %.1f us |' % (k, v['k1_us'], v['k2_us'], v['tick_us'])
                                            for k, v in row.items()) +
              '  a == b bitwise: %s, max |raw c - raw d| %.3g' % (same_ab, err_cd), flush=True)
        assert same_ab and err_cd < 1e-5, (same_ab, err_cd)
        results.append(dict(round=rep, arms=row, a_equals_b=same_ab, max_raw_diff_cd=err_cd))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(dict(card=gpu, streams=S, results=results), f, indent=1)


if __name__ == '__main__':
    main()
