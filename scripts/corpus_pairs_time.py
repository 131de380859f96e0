"""Pool models over chosen recordings (DESIGN.md §3 "Pool models over chosen recordings", §6).

k pool models whose slots cycle over 64 seeded default-shaped networks (H = 20 over 13 MFCCs).  Arms, alternated in every
round after a warm-up round, CUDA events around each arm's calls:
  (a) owner clips: k models x 64 clips of 1-5 s each (model i owns clips 64 i .. 64 i + 63), listener c = 1024 and
      simulate c = 4096.  pairs: one pb_score_corpus_pairs call over the k x 64 (model, own clip) pairs, reductions only.
      pool: one pb_score_corpus_pool call per model over its own 64 clips, reductions only.
  (b) cross product as pairs: a 1 h corpus x k models, both schedules.  pairs: the model-major cross product as a pair
      list; pool: one pb_score_corpus_pool call.  Reductions only.
  (c) mining: a 100 h corpus x k models, listener c = 2048.  pairs: the cross product with hits only (d_n_hits and room
      for every hit, up to 2^26 of them); pool: pb_score_corpus_pool with activations only (per_window=False).
Reported per arm: lowest-highest ms over the rounds, profile slot 0 (K1) and slot 1 (scans, trigger and hit passes) ms, and
pair-windows per second of slot 1.  Checked every round: (a) and (b) the arms' reductions are bit-identical; (c) the hit
count is the same in every round, and one untimed pairs call with activations equals the pool arm's activations.

    python scripts/corpus_pairs_time.py [--k 1024] [--rounds 3] [--mining-hours 100] [--out result.json]
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
CLIPS = 64


def owner_clips(k, seed=1):
    """k * CLIPS clips of 1-5 s (multiples of 8 samples), seeded noise on the device."""
    rs = np.random.RandomState(seed)
    lens = (rs.uniform(1, 5, k * CLIPS) * SR).astype(np.int64) & ~7
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    g = torch.Generator(device='cuda').manual_seed(seed)
    pcm = (torch.randn(int(offs[-1]), generator=g, device='cuda') * 3000).clamp_(-32768, 32767).to(torch.int16)
    return pcm, offs


def red_bufs(n, sched):
    f = lambda dt: torch.empty(n, dtype=dt, device='cuda')
    return {'activations': f(torch.int64), 'above': f(torch.int64) if sched else None, 'sum': f(torch.float64) if sched else None}


def timed(pool, fn):
    pool.profile(True)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    out = fn()
    t1.record()
    torch.cuda.synchronize()
    prof = np.asarray(pool.profile_read()[0][:2])
    pool.profile(False)
    return t0.elapsed_time(t1), prof, out


def pairs_call(pool, pcm, offs, models, recs, sched, c, red=None, hits=None):
    """red: reduction buffers [n_pairs]; hits: (d_hits, capacity, d_n_hits)."""
    red = red or {}
    d_hits, cap, d_n = hits if hits else (None, 0, None)
    check(pool.lib.pb_score_corpus_pairs(pool._h, _ptr(pcm), _np_ptr(offs), len(offs) - 1, _np_ptr(models), _np_ptr(recs),
                                         len(models), 32768, sched, c, 0.5, None, None, None, _ptr(red.get('activations')),
                                         _ptr(red.get('above')), _ptr(red.get('sum')), 0.5, _ptr(d_hits), cap, _ptr(d_n),
                                         pool._stream()))


def pool_call(pool, pcm, offs, ids, sched, c, red):
    check(pool.lib.pb_score_corpus_pool(pool._h, _ptr(pcm), _np_ptr(offs), len(offs) - 1, _np_ptr(ids), len(ids), 32768, sched,
                                        c, 0.5, None, None, None, _ptr(red['activations']), _ptr(red['above']),
                                        _ptr(red['sum']), pool._stream()))


def summary(times, profs, windows):
    t, p = np.asarray(times), np.asarray(profs)
    return dict(ms=[float(t.min()), float(t.max())], slot0_ms=[float(p[:, 0].min()), float(p[:, 0].max())],
                slot1_ms=[float(p[:, 1].min()), float(p[:, 1].max())],
                pair_windows_per_s_slot1=[windows / (p[:, 1].max() / 1e3), windows / (p[:, 1].min() / 1e3)])


def run_arms(rounds, arms, check_same):
    """arms: name -> fn() returning (ms, prof, outputs).  Round 0 warms up."""
    times = {a: [] for a in arms}
    profs = {a: [] for a in arms}
    same = True
    for rnd in range(rounds + 1):
        outs = {}
        for a, fn in arms.items():
            ms, prof, outs[a] = fn()
            if rnd:
                times[a].append(ms)
                profs[a].append(prof)
        same &= check_same(outs)
        print('round', rnd, {a: round(times[a][-1], 2) for a in arms} if rnd else 'warm-up', flush=True)
    return times, profs, bool(same)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--k', type=int, default=1024)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--cross-hours', type=float, default=1.0)
    ap.add_argument('--mining-hours', type=float, default=100.0)
    ap.add_argument('--mining-rounds', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    k = args.k
    res = dict(card=card(), k=k, rounds=args.rounds, runs=[])
    nets = [m.GruModel.random(13, 20, seed=1000 + i, scale=0.1) for i in range(NETS)]
    pool = m.PreciseB200()
    pool.set_pool(k)
    for i in range(k):
        pool.pool_load(i, nets[i % NETS])
    ids = np.arange(k, dtype=np.int32)

    def same_red(outs):
        a, b = outs['pairs'], outs['pool']
        return all(a[x] is None or np.array_equal(a[x], b[x]) for x in a)

    # (a) owner clips
    pcm, offs = owner_clips(k)
    models = np.repeat(ids, CLIPS).astype(np.int32)
    recs = np.arange(k * CLIPS, dtype=np.int32)
    for name, c in (('listener', 1024), ('simulate', 4096)):
        s = 0 if name == 'listener' else 1
        Wp = sum(pool.corpus_windows(int(L), name, c) for L in np.diff(offs))

        def arm_pairs():
            red = red_bufs(len(models), s)
            ms, prof, _ = timed(pool, lambda: pairs_call(pool, pcm, offs, models, recs, s, c, red))
            return ms, prof, {x: None if v is None else v.cpu().numpy() for x, v in red.items()}

        def arm_pool():
            red = red_bufs(len(models), s)
            def calls():
                for i in range(k):
                    a, b = offs[i * CLIPS], offs[(i + 1) * CLIPS]
                    r = {x: None if v is None else v[i * CLIPS:(i + 1) * CLIPS] for x, v in red.items()}
                    pool_call(pool, pcm[a:b], offs[i * CLIPS:(i + 1) * CLIPS + 1] - a, ids[i:i + 1], s, c, r)
            ms, prof, _ = timed(pool, calls)
            return ms, prof, {x: None if v is None else v.cpu().numpy() for x, v in red.items()}

        times, profs, same = run_arms(args.rounds, {'pairs': arm_pairs, 'pool': arm_pool}, same_red)
        run = dict(test='owner clips', schedule=name, chunk=c, pairs=len(models), hours=float(offs[-1]) / SR / 3600,
                   pair_windows=Wp, outputs_identical=same, arms={a: summary(times[a], profs[a], Wp) for a in times})
        res['runs'].append(run)
        print(json.dumps(run), flush=True)
    del pcm
    torch.cuda.empty_cache()

    # (b) cross product as pairs
    pcm, offs = corpus(args.cross_hours)
    n_rec = len(offs) - 1
    models = np.repeat(ids, n_rec).astype(np.int32)
    recs = np.tile(np.arange(n_rec, dtype=np.int32), k)
    for name, c in (('listener', 1024), ('simulate', 4096)):
        s = 0 if name == 'listener' else 1
        W = sum(pool.corpus_windows(int(L), name, c) for L in np.diff(offs))

        def arm_pairs():
            red = red_bufs(k * n_rec, s)
            ms, prof, _ = timed(pool, lambda: pairs_call(pool, pcm, offs, models, recs, s, c, red))
            return ms, prof, {x: None if v is None else v.cpu().numpy() for x, v in red.items()}

        def arm_pool():
            red = red_bufs(k * n_rec, s)
            ms, prof, _ = timed(pool, lambda: pool_call(pool, pcm, offs, ids, s, c, red))
            return ms, prof, {x: None if v is None else v.cpu().numpy() for x, v in red.items()}

        times, profs, same = run_arms(args.rounds, {'pairs': arm_pairs, 'pool': arm_pool}, same_red)
        run = dict(test='cross product', schedule=name, chunk=c, pairs=len(models), hours=float(offs[-1]) / SR / 3600,
                   pair_windows=k * W, outputs_identical=same, arms={a: summary(times[a], profs[a], k * W) for a in times})
        res['runs'].append(run)
        print(json.dumps(run), flush=True)
    del pcm
    torch.cuda.empty_cache()

    # (c) mining, listener c = 2048
    pcm, offs = corpus(args.mining_hours)
    n_rec = len(offs) - 1
    models = np.repeat(ids, n_rec).astype(np.int32)
    recs = np.tile(np.arange(n_rec, dtype=np.int32), k)
    c = 2048
    W = sum(pool.corpus_windows(int(L), 'listener', c) for L in np.diff(offs))
    d_n = torch.zeros(1, dtype=torch.int64, device='cuda')
    pairs_call(pool, pcm, offs, models, recs, 0, c, hits=(None, 0, d_n))
    total = int(d_n.item())
    cap = min(total, 1 << 26)                                   # room for every hit up to 512 MB of them
    d_hits = torch.empty(max(cap, 1), dtype=torch.int64, device='cuda')

    def arm_pairs():
        ms, prof, _ = timed(pool, lambda: pairs_call(pool, pcm, offs, models, recs, 0, c, hits=(d_hits, cap, d_n)))
        return ms, prof, int(d_n.item())

    pool_act = {}

    def arm_pool():
        red = red_bufs(k * n_rec, 0)
        ms, prof, _ = timed(pool, lambda: pool_call(pool, pcm, offs, ids, 0, c, red))
        pool_act['a'] = red['activations'].cpu().numpy()
        return ms, prof, None

    times, profs, same = run_arms(args.mining_rounds, {'pairs': arm_pairs, 'pool': arm_pool},
                                  lambda outs: outs['pairs'] == total)
    red = red_bufs(k * n_rec, 0)
    pairs_call(pool, pcm, offs, models, recs, 0, c, red, hits=(None, 0, d_n))
    same &= bool(np.array_equal(red['activations'].cpu().numpy(), pool_act['a'])) and int(d_n.item()) == total
    run = dict(test='mining', schedule='listener', chunk=c, pairs=len(models), hours=float(offs[-1]) / SR / 3600,
               pair_windows=k * W, hits=total, hit_capacity=cap, outputs_identical=bool(same),
               arms={a: summary(times[a], profs[a], k * W) for a in times})
    res['runs'].append(run)
    print(json.dumps(run), flush=True)
    pool.close()
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
