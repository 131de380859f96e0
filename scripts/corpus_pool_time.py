"""Pool models over recorded corpora (DESIGN.md §3 "Pool models over a recorded corpus", §6).

Seeded on-device corpora as corpus_time.py builds them (1 h and 100 h) and k pool models whose slots cycle over 64 seeded
default-shaped networks (H = 20 over 13 MFCCs), both schedules (listener c = 1024, simulate c = 4096).  Arms:
  a      one handle per group of 8 models as a bank (8 handles, reused cyclically: the slots cycle with period 64), one
         pb_score_corpus per group with raw and the reductions; CUDA events around the k / 8 calls only
  b      one pool handle, pb_score_corpus_pool with the reductions only
  b-raw  b with d_raw, where k W floats fit in 24 GB
  nmN-o  b with N models per CTA and grid order o (1: model groups vary fastest, 0: window tiles), pb_debug_corpus_pool_scan;
         above --variant-pairs (model, window) pairs only the --large-variants
Reported per arm: lowest-highest call ms over ROUNDS alternating rounds, hours of audio x models per device second, profile
slot 0 (K1) and slot 1 (scans and trigger) ms, (model, window) pairs per second, and for the pool arms the scan's byte
model: fragment bytes per (tile, group) plus 1 856 B of rows per window per group, over slot 1.  Checked every round:
the reductions (activations, and above / sum for simulate) of a and of every b arm are bit-identical.

    python scripts/corpus_pool_time.py [--hours 1 100] [--k 64 1024] [--rounds 4] [--out result.json]
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
from mycroft_precise_b200.core import _np_ptr, _ptr, check   # noqa: E402
from bank_time import card              # noqa: E402
from corpus_time import SR, corpus      # noqa: E402

NETS = 64
FRAG = 14208                             # bytes of one model's fragments, loaded once per CTA
ROW_BYTES = 29 * 64                      # one window's rows: n_features rows of 16 floats
DEFAULT_NM = 1                           # CORPUS_POOL_NM


def nets():
    return [m.GruModel.random(13, 20, seed=1000 + i, scale=0.1) for i in range(NETS)]


def bank_handles(models):
    out = []
    for b in range(NETS // 8):
        core = m.PreciseB200()
        g = models[8 * b]
        core.load_weights(g.kernel, g.recurrent, g.bias, g.dense_w, g.dense_b)
        for j in range(1, 8):
            core.add_model(models[8 * b + j])
        out.append(core)
    return out


def events():
    return torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)


def arm_a(banks, pcm, offs, k, sched, c, W, n_rec):
    """k / 8 bank calls; returns (ms, reductions [k][n_rec] per key)."""
    s = 0 if sched == 'listener' else 1
    raw = torch.empty((8, W), dtype=torch.float32, device='cuda')
    red = {'activations': torch.empty((k, n_rec), dtype=torch.int64, device='cuda')}
    if s:
        red['above'] = torch.empty((k, n_rec), dtype=torch.int64, device='cuda')
        red['sum'] = torch.empty((k, n_rec), dtype=torch.float64, device='cuda')
    for b in banks:
        b.profile(True)
    t0, t1 = events()
    t0.record()
    for g in range(k // 8):
        b = banks[g % len(banks)]
        sl = lambda key: _ptr(red[key][8 * g:8 * g + 8]) if key in red else None
        check(b.lib.pb_score_corpus(b._h, _ptr(pcm), _np_ptr(offs), n_rec, 32768, s, c, 0.5, _ptr(raw), None, None,
                                    sl('activations'), sl('above'), sl('sum'), b._stream()))
    t1.record()
    torch.cuda.synchronize()
    prof = np.zeros(2)
    for b in banks:
        prof += np.asarray(b.profile_read()[0][:2])
        b.profile(False)
    return t0.elapsed_time(t1), prof, {key: v.cpu().numpy() for key, v in red.items()}


def arm_b(pool, pcm, offs, ids, sched, c, W, n_rec, with_raw):
    """One pool call with the reductions, and raw [k][W] when with_raw."""
    s = 0 if sched == 'listener' else 1
    k = len(ids)
    raw = torch.empty((k, W), dtype=torch.float32, device='cuda') if with_raw else None
    red = {'activations': torch.empty((k, n_rec), dtype=torch.int64, device='cuda')}
    if s:
        red['above'] = torch.empty((k, n_rec), dtype=torch.int64, device='cuda')
        red['sum'] = torch.empty((k, n_rec), dtype=torch.float64, device='cuda')
    pool.profile(True)
    t0, t1 = events()
    t0.record()
    check(pool.lib.pb_score_corpus_pool(pool._h, _ptr(pcm), _np_ptr(offs), n_rec, _np_ptr(ids), k, 32768, s, c, 0.5, _ptr(raw),
                                        None, None, _ptr(red['activations']), _ptr(red.get('above')), _ptr(red.get('sum')),
                                        pool._stream()))
    t1.record()
    torch.cuda.synchronize()
    prof = np.asarray(pool.profile_read()[0][:2])
    pool.profile(False)
    del raw
    return t0.elapsed_time(t1), prof, {key: v.cpu().numpy() for key, v in red.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--hours', type=float, nargs='+', default=[1.0, 100.0])
    ap.add_argument('--k', type=int, nargs='+', default=[64, 1024])
    ap.add_argument('--rounds', type=int, default=4)
    ap.add_argument('--variants', default='1-1,1-0,2-1,2-0,4-1,4-0,8-1,8-0')
    ap.add_argument('--variant-pairs', type=float, default=1e9, help='above this many (model, window) pairs, run --large-variants')
    ap.add_argument('--large-variants', default='1-1,1-0,2-1,2-0')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    res = dict(card=card(), rounds=args.rounds, runs=[])
    models = nets()
    banks = bank_handles(models)
    variants = [tuple(int(x) for x in v.split('-')) for v in args.variants.split(',') if v]
    large = [tuple(int(x) for x in v.split('-')) for v in args.large_variants.split(',') if v]
    for hours in args.hours:
        pcm, offs = corpus(hours)
        n_rec = len(offs) - 1
        real_h = float(offs[-1]) / SR / 3600
        for k in args.k:
            pool = m.PreciseB200()
            pool.set_pool(k)
            for i in range(k):
                pool.pool_load(i, models[i % NETS])
            ids = np.arange(k, dtype=np.int32)
            for sched, c in (('listener', 1024), ('simulate', 4096)):
                W = sum(pool.corpus_windows(int(L), sched, c) for L in np.diff(offs))
                arms = ['a', 'b'] + (['b-raw'] if k * W * 4 <= 24 << 30 else []) + ['nm%d-%d' % v for v in (variants if k * W <= args.variant_pairs else large)]
                times = {a: [] for a in arms}
                profs = {a: [] for a in arms}
                identical = True
                for rnd in range(args.rounds + 1):                      # round 0 warms every shape up
                    ms, prof, ref = arm_a(banks, pcm, offs, k, sched, c, W, n_rec)
                    got = {'a': (ms, prof)}
                    for a in arms[1:]:
                        if a.startswith('nm'):
                            nm, order = (int(x) for x in a[2:].split('-'))
                            pool.corpus_pool_scan(nm, order)
                        ms, prof, red = arm_b(pool, pcm, offs, ids, sched, c, W, n_rec, a == 'b-raw')
                        pool.corpus_pool_scan(0, -1)
                        got[a] = (ms, prof)
                        identical &= all(np.array_equal(red[key], ref[key]) for key in ref)
                    print('round', rnd, k, sched, {a: round(got[a][0], 2) for a in arms}, flush=True)
                    if rnd:
                        for a in arms:
                            times[a].append(got[a][0])
                            profs[a].append(got[a][1])
                pairs = k * W
                run = dict(hours=real_h, recordings=n_rec, k=k, schedule=sched, chunk=c, windows=W,
                           reductions_identical=bool(identical), arms={})
                for a in arms:
                    t = np.asarray(times[a])
                    p = np.asarray(profs[a])
                    r = dict(ms=[float(t.min()), float(t.max())], slot0_ms=[float(p[:, 0].min()), float(p[:, 0].max())],
                             slot1_ms=[float(p[:, 1].min()), float(p[:, 1].max())],
                             hours_models_per_s=[real_h * k / (t.max() / 1e3), real_h * k / (t.min() / 1e3)],
                             pairs_per_s=[pairs / (t.max() / 1e3), pairs / (t.min() / 1e3)])
                    if a != 'a':
                        nm = int(a[2:].split('-')[0]) if a.startswith('nm') else DEFAULT_NM
                        groups = (k + nm - 1) // nm
                        scan_bytes = groups * (((W + 63) // 64) * nm * FRAG + W * ROW_BYTES)
                        r['scan_model_GB'] = scan_bytes / 1e9
                        r['scan_GBps_on_slot1'] = [scan_bytes / (p[:, 1].max() / 1e3) / 1e9,
                                                   scan_bytes / (p[:, 1].min() / 1e3) / 1e9]
                    run['arms'][a] = r
                res['runs'].append(run)
                print(json.dumps(run), flush=True)
            pool.close()
        del pcm
        torch.cuda.empty_cache()
    for b in banks:
        b.close()
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
