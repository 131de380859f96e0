"""The combined bank + pool tick at the bench size (DESIGN.md §3 "Combined bank + pool tick", §6).

131 072 streams, every stream on bank slot 0 (the default-shaped network, H = 20 over 13 MFCCs) and on one of 1 024 pool
models (128 streams each; the slots cycle over 64 distinct seeded networks, as in pool_time.py), seeded PCM.
  arm a: a bank handle's update_models plus a pool handle's update_pool per tick (two K1 passes);
  arm b: one handle with the same bank and pool, update_all (one K1);
  arm c: b with pool trigger settings on every stream (the models' own values, so the outputs stay bit-identical): the
         pool's scan writes raw and conf only and pool_trigger_kernel runs after it.
The arms alternate in one process (REPS rounds); each round primes PRIME untimed ticks and times TIMED: K1 / K2 from the
library's CUDA-event profile (slots 0 / 1, summed over an arm's handles), the tick from CUDA events around the timed loop.
raw, conf and fired must be bit-identical across the arms.

    python scripts/bank_pool_time.py [--out result.json]
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
from bank_time import S, PRIME, TIMED, card, timed   # noqa: E402
from pool_time import load_pool         # noqa: E402

N_POOL, REPS = 1024, 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='also write the results as JSON to this file')
    ap.add_argument('--reps', type=int, default=REPS, help='rounds of alternating arms')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bank_pool_time.py needs a CUDA device')
    gpu = card()
    print('card:', gpu, flush=True)
    models = []
    for i in range(64):
        g = m.GruModel.random(13, 20, seed=i, scale=0.1)
        g.dense_b = 3.0
        models.append(g)
    pcm = [torch.from_numpy(np.clip(np.random.RandomState(i).randn(S, 1024) * 3000, -32768, 32767).astype(np.int16)).cuda()
           for i in range(2)]
    assign = (np.arange(S) // (S // N_POOL)).astype(np.int32)
    bank = m.StreamBatch(models[0], S)
    pool = m.StreamBatch(models[0], S)
    load_pool(pool, N_POOL, models)
    pool.set_stream_pool(assign)
    both, trig = m.StreamBatch(models[0], S), m.StreamBatch(models[0], S)
    for sb in (both, trig):
        load_pool(sb, N_POOL, models)
        sb.set_stream_pool(assign)
    trig.set_stream_pool_trigger(0.5, 3, 2048)             # pool_load's defaults and 2 * chunk_samples: the models' own

    def tick_a(p):
        ob, op = bank.update_models(p), pool.update_pool(p)
        return {q: torch.cat([ob[q], op[q][None]]) for q in ('raw', 'conf', 'fired')}

    arms = [('a', [bank, pool], tick_a), ('b', [both], both.update_all), ('c', [trig], trig.update_all)]
    results = []
    for rep in range(args.reps):
        row, outs = {}, {}
        for name, handles, tick in arms:
            t, o = timed(handles, tick, pcm)
            outs[name] = {q: o[q].clone() for q in ('raw', 'conf', 'fired')}
            row[name] = t
            print('round %d  %s  K1 %7.1f us  K2 %7.1f us  tick %7.1f us' % (rep, name, t['k1_us'], t['k2_us'], t['tick_us']),
                  flush=True)
        same = lambda x, y: bool(torch.equal(x.contiguous().view(torch.uint8), y.contiguous().view(torch.uint8)))
        ok = all(same(outs['a'][q], outs[x][q]) for x in ('b', 'c') for q in ('raw', 'conf', 'fired'))
        fired = {k: [int(r) for r in v['fired'].sum(1)] for k, v in outs.items()}
        print('round %d  a / b / c bit-identical: %s, fired (bank, pool) per arm %s' % (rep, ok, fired), flush=True)
        assert ok
        results.append(dict(round=rep, fired=fired, **row))
    for name in ('a', 'b', 'c'):
        for key in ('k1_us', 'k2_us', 'tick_us'):
            v = [r[name][key] for r in results]
            print('%s %-7s min %7.1f  max %7.1f' % (name, key, min(v), max(v)))
    if args.out:
        with open(args.out, 'w') as fo:
            json.dump(dict(card=gpu, streams=S, pool_models=N_POOL, prime=PRIME, timed=TIMED, results=results), fo, indent=1)
    for sb in (bank, pool, both, trig):
        sb.core.close()


if __name__ == '__main__':
    main()
