"""Per-stream TriggerDetector settings at the bench size (DESIGN.md §3 "Per-stream trigger settings", §6).

131 072 streams, default-shaped networks (H = 20 over 13 MFCCs) with seeded weights and a dense bias of 3.0 (so that
streams fire), seeded PCM.
  arm a: a one-model handle without settings, update;
  arm b: the same model on a second handle with every stream set to the model's own values (the trigger kernel path);
  arm c: an 8-model routed bank, stream s subscribed to model s mod 8 only, without settings, update_models;
  arm d: arm c with every stream of every model set to the model's own values.
The arms alternate in one process (REPS rounds), each round primes PRIME untimed ticks and times TIMED: K1 / K2 from the
library's CUDA-event profile (slots 0 / 1), tick time from CUDA events around the timed loop.  Every arm sees the same tick
sequence, so the last tick's raw, conf, fired and the counts must be bit-identical between a and b and between c and d.

    python scripts/trigger_time.py [--out result.json]
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
    x, y = x.contiguous(), y.contiguous()
    return x.shape == y.shape and bool(torch.equal(x.view(torch.uint8), y.view(torch.uint8)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='also write the results as JSON to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('trigger_time.py needs a CUDA device')
    gpu = card()
    print('card:', gpu, flush=True)
    models = [m.GruModel.random(13, 20, seed=i, scale=0.1) for i in range(8)]
    for mod in models:
        mod.dense_b = 3.0                   # confidences near the default threshold, so that streams fire
    pcm = [torch.from_numpy(np.clip(np.random.RandomState(i).randn(S, 1024) * 3000, -32768, 32767).astype(np.int16)).cuda()
           for i in range(2)]
    a, b = m.StreamBatch(models[0], S), m.StreamBatch(models[0], S)
    b.set_stream_trigger(0, 0.5, 3, 2048)                  # StreamBatch's defaults: sensitivity 0.5, level 3, 1024 samples
    c, d = bank(models, S), bank(models, S)
    owner = (1 << (np.arange(S) % 8)).astype(np.uint8)
    for x in (c, d):
        x.set_stream_models(owner)
    for slot in range(8):
        d.set_stream_trigger(slot, 0.5, 3, 2048)
    arms = [('a', [a], a.update), ('b', [b], b.update), ('c', [c], c.update_models), ('d', [d], d.update_models)]
    results = []
    for rep in range(REPS):
        row, outs = {}, {}
        for name, handles, tick in arms:
            row[name], o = timed(handles, tick, pcm)
            outs[name] = {k: v.clone() for k, v in o.items()}
            print('round %d  %s  K1 %7.1f us  K2 %7.1f us  tick %7.1f us'
                  % (rep, name, row[name]['k1_us'], row[name]['k2_us'], row[name]['tick_us']), flush=True)
        ab = all(same_bits(outs['a'][k], outs['b'][k]) for k in ('raw', 'conf', 'fired')) and same_bits(a.count, b.count)
        cd = all(same_bits(outs['c'][k], outs['d'][k]) for k in ('raw', 'conf', 'fired')) and same_bits(c.counts, d.counts)
        print('round %d  a/b last tick and count bit-identical: %s, c/d: %s (counts a %d, c %s)'
              % (rep, ab, cd, int(a.count.item()), c.counts.cpu().tolist()), flush=True)
        assert ab and cd
        results.append(dict(round=rep, **row))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(dict(card=gpu, streams=S, prime=PRIME, timed=TIMED, results=results), f, indent=1)
    for x in (a, b, c, d):
        x.core.close()


if __name__ == '__main__':
    main()
