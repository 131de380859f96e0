"""The model pool at the bench size (DESIGN.md §3 "Model pool", §6).

131 072 streams, default-shaped networks (H = 20 over 13 MFCCs, Keras's default activations) with seeded weights and a dense
bias that makes them fire, seeded PCM.  Pool slots cycle over 64 distinct networks: every slot is its own copy in the pool's
fragment array, so a tick loads what distinct networks would.
  arm a: one-model handle, update;
  arm b: pool, every stream on one model (block tiles only);
  arm c: 1 024 models x 128 streams (block tiles);
  arms b-warp, c-warp: b and c with every position in warp tiles (pb_debug_pool_tiles);
  arm d: 32 768 models x 4 streams (warp tiles);
  arm e: 131 072 models x 1 stream (1.86 GB of fragments; load time not measured);
  arm f: an 8-model routed bank, stream s on model s mod 8 (f-bank), against a pool with the same 8 models and assignment
         (f-pool).
The arms alternate in one process (REPS rounds); each round primes PRIME untimed ticks and times TIMED: K1 / K2 from the
library's CUDA-event profile (slots 0 / 1), the tick from CUDA events around the timed loop.  raw, conf and fired must be
bit-identical between a and b, between b / c and their warp-tile arms, and between f-bank's subscribed rows and f-pool.

Byte model of a pool tick's K2: 14 208 B of fragments per block tile and per warp tile, plus 1 856 B of ring rows (29 rows of
16 floats) per item, against the H100 SXM data-sheet 3.35 TB/s.

    python scripts/pool_time.py [--out result.json]
"""
import argparse
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np                      # noqa: E402
import torch                            # noqa: E402
import mycroft_precise_b200 as m        # noqa: E402
from mycroft_precise_b200.core import check   # noqa: E402
from bank_time import S, PRIME, TIMED, REPS, card, timed   # noqa: E402

FRAG, ROWS, PEAK = 14208, 29 * 16 * 4, 3.35e12


def load_pool(sb, n_models, models):
    """Slot i gets models[i % len(models)], through the C ABI (the Python layer's checks, once per distinct network)."""
    core = sb.core
    core.set_pool(n_models)
    args = [core._model_args(g, None, 0.5, 3, False, core._pool_cdf) for g in models]
    for i in range(n_models):
        cfg, (k, u, b, w, bd), cd = args[i % len(args)]
        vp = lambda a: a.ctypes.data_as(C.c_void_p)
        check(core.lib.pb_pool_load(core._h, i, C.byref(cfg), vp(k), vp(u), vp(b), vp(w), bd,
                                    None if cd is None else vp(cd), 0 if cd is None else len(cd)))


def tiles(group, n_groups):
    """(block tiles, warp tiles) of n_groups models of `group` streams each."""
    return n_groups * (group // 64), n_groups * (-(-(group % 64) // 16))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='also write the results as JSON to this file')
    ap.add_argument('--reps', type=int, default=REPS, help='rounds of alternating arms')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('pool_time.py needs a CUDA device')
    gpu = card()
    print('card:', gpu, flush=True)
    models = []
    for i in range(64):
        g = m.GruModel.random(13, 20, seed=i, scale=0.1)
        g.dense_b = 3.0
        models.append(g)
    pcm = [torch.from_numpy(np.clip(np.random.RandomState(i).randn(S, 1024) * 3000, -32768, 32767).astype(np.int16)).cuda()
           for i in range(2)]
    a = m.StreamBatch(models[0], S)
    arms = [('a', a, a.update, (0, 0))]
    for name, group in (('b', S), ('b-warp', S), ('c', 128), ('c-warp', 128), ('d', 4), ('e', 1)):
        sb = m.StreamBatch(models[0], S)
        n = S // group
        load_pool(sb, n, models)
        sb.set_stream_pool((np.arange(S) // group).astype(np.int32))
        tl = tiles(group, n)
        if name.endswith('-warp'):
            check(sb.core.lib.pb_debug_pool_tiles(sb.core._h, 1))
            tl = (0, n * -(-group // 16))
        arms.append((name, sb, sb.update_pool, tl))
        print('arm %s loaded: %d models x %d streams' % (name, n, group), flush=True)
    owner = (np.arange(S) % 8).astype(np.int32)
    fb = m.StreamBatch(models[0], S)
    for g in models[1:8]:
        fb.add_model(g)
    fb.set_stream_models((1 << owner).astype(np.uint8))
    fp = m.StreamBatch(models[0], S)
    load_pool(fp, 8, models[:8])
    fp.set_stream_pool(owner)
    arms += [('f-bank', fb, fb.update_models, None), ('f-pool', fp, fp.update_pool, tiles(S // 8, 8))]
    sel = torch.from_numpy(owner).long().cuda()
    cols = torch.arange(S, device='cuda')
    results = []
    for rep in range(args.reps):
        row, outs = {}, {}
        for name, sb, tick, tl in arms:
            t, o = timed([sb], tick, pcm)
            outs[name] = {q: o[q].clone() for q in ('raw', 'conf', 'fired')}
            if tl is not None and name != 'a':
                nbytes = (tl[0] + tl[1]) * FRAG + S * ROWS
                t.update(block_tiles=tl[0], warp_tiles=tl[1], k2_bytes=nbytes, k2_tbs=nbytes / (t['k2_us'] * 1e-6) / 1e12,
                         k2_share_of_peak=nbytes / PEAK / (t['k2_us'] * 1e-6))
            row[name] = t
            print('round %d  %-7s K1 %7.1f us  K2 %8.1f us  tick %8.1f us%s'
                  % (rep, name, t['k1_us'], t['k2_us'], t['tick_us'],
                     '  K2 bytes %.3g (%.2f TB/s, %.0f %% of 3.35)' % (t['k2_bytes'], t['k2_tbs'], 100 * t['k2_share_of_peak'])
                     if 'k2_bytes' in t else ''), flush=True)
        same = lambda x, y: bool(torch.equal(x.contiguous().view(torch.uint8), y.contiguous().view(torch.uint8)))
        ab = all(same(outs['a'][q], outs['b'][q]) for q in ('raw', 'conf', 'fired'))
        f = all(same(outs['f-bank'][q][sel, cols], outs['f-pool'][q]) for q in ('raw', 'conf', 'fired'))
        warp = all(same(outs[x][q], outs[x + '-warp'][q]) for x in ('b', 'c') for q in ('raw', 'conf', 'fired'))
        fired = {k: int(v['fired'].sum()) for k, v in outs.items()}
        print('round %d  a/b bit-identical: %s, b / c against their warp-tile arms: %s, f-bank subscribed rows / f-pool '
              'bit-identical: %s, fired per arm %s' % (rep, ab, warp, f, fired), flush=True)
        assert ab and warp and f
        results.append(dict(round=rep, fired=fired, **row))
    if args.out:
        with open(args.out, 'w') as fo:
            json.dump(dict(card=gpu, streams=S, prime=PRIME, timed=TIMED, results=results), fo, indent=1)
    for _, sb, _, _ in arms:
        sb.core.close()


if __name__ == '__main__':
    main()
