"""Per-stream model subscriptions at the bench size (DESIGN.md §3 "Per-stream model subscriptions", §6).

131 072 streams, default-shaped networks (H = 20 over 13 MFCCs) with seeded weights, seeded PCM.
  arm a: an 8-model bank, unrouted, update_models;
  arm b: the same bank on a routed handle, stream s subscribed to model s mod 8 only;
  arm c: one model on a one-model handle, update;
  arm d: a 2-model bank, routed with every stream subscribed to both (d-routed), beside the unrouted 2-model bank (d-bank).
The arms alternate in one process (REPS rounds), each round primes PRIME untimed ticks and times TIMED: K1 / K2 from the
library's CUDA-event profile (slots 0 / 1), tick time from CUDA events around the timed loop.  Every arm sees the same tick
sequence, so subscribed raw outputs must be bit-identical between a and b and between the two halves of d.

    python scripts/route_time.py [--out result.json]
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
from bank_time import S, PRIME, TIMED, REPS, card, timed   # noqa: E402


def bank(models, S):
    sb = m.StreamBatch(models[0], S)
    for mod in models[1:]:
        sb.add_model(mod)
    return sb


def same_bits(x, y):
    return bool(torch.equal(x.contiguous().view(torch.int32), y.contiguous().view(torch.int32)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='also write the results as JSON to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('route_time.py needs a CUDA device')
    gpu = card()
    print('card:', gpu, flush=True)
    models = [m.GruModel.random(13, 20, seed=i, scale=0.1) for i in range(8)]
    pcm = [torch.from_numpy(np.clip(np.random.RandomState(i).randn(S, 1024) * 3000, -32768, 32767).astype(np.int16)).cuda()
           for i in range(2)]
    a, b = bank(models, S), bank(models, S)
    owner = np.arange(S) % 8
    b.set_stream_models((1 << owner).astype(np.uint8))
    c = m.StreamBatch(models[0], S)
    d_bank, d_routed = bank(models[:2], S), bank(models[:2], S)
    d_routed.set_stream_models(np.full(S, 0x03, np.uint8))
    arms = [('a', [a], a.update_models), ('b', [b], b.update_models), ('c', [c], c.update),
            ('d-bank', [d_bank], d_bank.update_models), ('d-routed', [d_routed], d_routed.update_models)]
    sel = torch.from_numpy(owner).cuda()
    results = []
    for rep in range(REPS):
        row, outs = {}, {}
        for name, handles, tick in arms:
            row[name], o = timed(handles, tick, pcm)
            outs[name] = o['raw'].clone()
            print('round %d  %-8s K1 %7.1f us  K2 %7.1f us  tick %7.1f us'
                  % (rep, name, row[name]['k1_us'], row[name]['k2_us'], row[name]['tick_us']), flush=True)
        ra, rb = outs['a'], outs['b']
        ab = all(same_bits(ra[i][sel == i], rb[i][sel == i]) for i in range(8))
        unsub = all(bool(torch.isnan(rb[i][sel != i]).all()) for i in range(8))
        dd = same_bits(outs['d-bank'], outs['d-routed'])
        print('round %d  a/b subscribed raw bit-identical: %s, b unsubscribed all NaN: %s, d halves bit-identical: %s'
              % (rep, ab, unsub, dd), flush=True)
        assert ab and unsub and dd
        results.append(dict(round=rep, **row))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(dict(card=gpu, streams=S, prime=PRIME, timed=TIMED, results=results), f, indent=1)
    for x in (a, b, c, d_bank, d_routed):
        x.core.close()


if __name__ == '__main__':
    main()
