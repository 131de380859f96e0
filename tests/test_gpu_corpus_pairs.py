"""Pool models over chosen recordings (pb_score_corpus_pairs, offline.score_corpus_pairs / simulate_pairs /
false_activations_pool).  The reference for every pair is the slice of its recording in the row pb_score_corpus_pool writes
for its model over the same recordings: every output must be equal bit for bit.  -m gpu except the null-handle checks."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle.trigger import OracleTrigger
from test_gpu_corpus_pool import _noise, _oracle_listener, _same, corpus, pool_models

gpu = pytest.mark.gpu
KEYS = ('raw', 'conf', 'fired', 'activations', 'above', 'sum')
WIN = ('raw', 'conf', 'fired')
CONFIGS = [('listener', 1024), ('listener', 2048), ('simulate', 4096), ('simulate', 1600)]


def _mod():
    import mycroft_precise_b200 as m
    return m


class Fixture:
    def __init__(self):
        import torch
        m = _mod()
        self.m = m
        self.spec = pool_models(m)
        self.recs, pcm, self.offsets = corpus()
        self.n_rec = len(self.recs)
        self.pcm = torch.from_numpy(pcm).cuda()
        self.pool = m.PreciseB200()
        self.pool.set_pool(len(self.spec))
        for i, (model, pr, sens, lvl) in enumerate(self.spec):
            self.pool.pool_load(i, model, pr, sensitivity=sens, trigger_level=lvl)
        self._ref = {}

    def ref(self, schedule, chunk, divisor=32768, pcm=None, offsets=None):
        """(host rows of score_corpus_pool over every model, window offsets of the recordings)."""
        key = (schedule, chunk, divisor, None if offsets is None else offsets.tobytes())
        if key not in self._ref:
            pcm = self.pcm if pcm is None else pcm
            offsets = self.offsets if offsets is None else offsets
            ids = np.arange(len(self.spec), dtype=np.int32)
            r = self.pool.score_corpus_pool(pcm, offsets, ids, schedule, chunk, 0.5, divisor)
            counts = [self.pool.corpus_windows(int(L), schedule, chunk) for L in np.diff(offsets)]
            wo = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
            self._ref[key] = ({k: None if r[k] is None else r[k].cpu().numpy() for k in KEYS}, wo)
        return self._ref[key]

    def close(self):
        self.pool.close()


@pytest.fixture(scope='module')
def fx():
    pytest.importorskip('torch')
    f = Fixture()
    yield f
    f.close()


def _host(res):
    return {k: None if res[k] is None else res[k].cpu().numpy() for k in KEYS}


def _check_pairs(got, ref, models, recs, keys=KEYS):
    """Every pair's outputs against the slice of the cross product; pair_offsets against the recordings' counts."""
    rows, wo = ref
    P = np.concatenate([[0], np.cumsum([wo[r + 1] - wo[r] for r in recs])]).astype(np.int64)
    if 'pair_offsets' in got:
        assert np.array_equal(got['pair_offsets'], P)
    for k in keys:
        if rows[k] is None:
            assert got[k] is None, k
            continue
        if got[k] is None:
            continue
        if k in WIN:
            assert got[k].shape == (P[-1],), k
            for p, (mid, r) in enumerate(zip(models, recs)):
                assert _same(got[k][P[p]:P[p + 1]], rows[k][mid][wo[r]:wo[r + 1]]), (k, p, mid, r)
        else:
            assert got[k].shape == (len(models),), k
            want = np.asarray([rows[k][mid][r] for mid, r in zip(models, recs)], rows[k].dtype)
            assert _same(got[k], want), k


def _pairs(fx, models, recs, schedule, chunk, divisor=32768, **kw):
    models, recs = np.asarray(models, np.int32), np.asarray(recs, np.int32)
    res = fx.pool.score_corpus_pairs(fx.pcm, fx.offsets, models, recs, schedule, chunk, 0.5, divisor, **kw)
    out = _host(res)
    out['pair_offsets'] = res['pair_offsets']
    if 'hits' in res:
        out['hits'] = res['hits'].cpu().numpy()
    return out


@gpu
@pytest.mark.parametrize('schedule,chunk', CONFIGS)
@pytest.mark.parametrize('divisor', [32768, 32767])
def test_cross_product_as_pairs(fx, schedule, chunk, divisor):
    M = len(fx.spec)
    models = np.repeat(np.arange(M), fx.n_rec)
    recs = np.tile(np.arange(fx.n_rec), M)
    got = _pairs(fx, models, recs, schedule, chunk, divisor)
    _check_pairs(got, fx.ref(schedule, chunk, divisor), models, recs)
    assert got['activations'].sum() > 0


LISTS = [
    # unsorted, repeated pairs, interleaved activation classes (2, 5, 8, 11 use tanh / sigmoid)
    ([3, 2, 0, 5, 3, 11, 8, 3, 1, 2], [8, 8, 4, 8, 2, 5, 7, 8, 6, 3]),
    # empty recording 0, recording 1 shorter than a window, recordings no pair names
    ([7, 7, 4, 0, 9, 6], [0, 1, 0, 8, 8, 1]),
    ([10], [8]),
    ([4, 4, 4, 4], [8, 8, 8, 8]),
]


@gpu
@pytest.mark.parametrize('schedule,chunk', [CONFIGS[0], CONFIGS[2]])
def test_routed_lists(fx, schedule, chunk):
    ref = fx.ref(schedule, chunk)
    for models, recs in LISTS:
        got = _pairs(fx, models, recs, schedule, chunk)
        _check_pairs(got, ref, models, recs)


@gpu
@pytest.mark.parametrize('schedule,chunk', [CONFIGS[0], CONFIGS[2]])
def test_tile_packing(fx, schedule, chunk):
    """60 clips of 1-3 s (under 64 windows each), five pairs per model: pairs in model runs (tiles cover several clips),
    then the same pairs interleaved so that consecutive pairs never share a model (one pair per tile).  Identical up to the
    permutation, and equal to the cross product's slices."""
    import torch
    rs = np.random.RandomState(5)
    clips = [_noise(int(rs.randint(16000, 48000)), 300 + i) for i in range(60)]
    offs = np.concatenate([[0], np.cumsum([len(c) for c in clips])]).astype(np.int64)
    pcm = torch.from_numpy(np.concatenate(clips)).cuda()
    M = len(fx.spec)
    models = np.repeat(np.arange(M), 5)
    recs = (np.arange(M * 5) * 7) % 60
    runs = fx.pool.score_corpus_pairs(pcm, offs, models.astype(np.int32), recs.astype(np.int32), schedule, chunk)
    perm = np.arange(M * 5).reshape(M, 5).T.reshape(-1)                  # model varies fastest
    inter = fx.pool.score_corpus_pairs(pcm, offs, models[perm].astype(np.int32), recs[perm].astype(np.int32), schedule, chunk)
    Pa, Pb = runs['pair_offsets'], inter['pair_offsets']
    assert (np.diff(Pa) < 64).all() and np.diff(Pa).sum() > 64
    a, b = _host(runs), _host(inter)
    for k in KEYS:
        if a[k] is None:
            continue
        for j, p in enumerate(perm):
            if k in WIN:
                assert _same(b[k][Pb[j]:Pb[j + 1]], a[k][Pa[p]:Pa[p + 1]]), (k, j)
            else:
                assert _same(b[k][j:j + 1], a[k][p:p + 1]), (k, j)
    a['pair_offsets'] = Pa
    _check_pairs(a, fx.ref(schedule, chunk, pcm=pcm, offsets=offs), models, recs)


@gpu
@pytest.mark.parametrize('schedule,chunk', [CONFIGS[0], CONFIGS[2]])
def test_batches(fx, schedule, chunk):
    """Batches of at most 1, 37 and 500 pair-windows (boundaries inside model runs; a pair larger than the cap forms its own
    batch), with the caller's d_raw and with raw in the handle's buffer (per_window=False, hits)."""
    models = [0, 0, 0, 5, 5, 2, 2, 2, 9, 9, 9, 9, 1]
    recs = [8, 4, 3, 8, 0, 5, 4, 8, 2, 3, 4, 8, 7]
    ref = fx.ref(schedule, chunk)
    hit = dict(hit_threshold=0.5) if schedule == 'listener' else {}
    full = _pairs(fx, models, recs, schedule, chunk, **hit)
    _check_pairs(full, ref, models, recs)
    try:
        for cap in (1, 37, 500):
            fx.pool.corpus_pairs_batch(cap)
            got = _pairs(fx, models, recs, schedule, chunk, **hit)
            _check_pairs(got, ref, models, recs)
            red = _pairs(fx, models, recs, schedule, chunk, per_window=False, **hit)
            assert red['raw'] is None and red['conf'] is None and red['fired'] is None
            _check_pairs(red, ref, models, recs)
            if hit:
                assert np.array_equal(got['hits'], full['hits']) and np.array_equal(red['hits'], full['hits'])
    finally:
        fx.pool.corpus_pairs_batch(0)


def _raw_call(fx, models, recs, thr, cap, hits_t=None, conf_t=None, schedule=0, chunk=1024):
    import torch
    models, recs = np.asarray(models, np.int32), np.asarray(recs, np.int32)
    n_hits = torch.full((1,), -7, dtype=torch.int64, device='cuda')
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    rc = fx.pool.lib.pb_score_corpus_pairs(fx.pool._h, p(fx.pcm), fx.offsets.ctypes.data_as(C.c_void_p), fx.n_rec,
                                           models.ctypes.data_as(C.c_void_p), recs.ctypes.data_as(C.c_void_p), len(models),
                                           32768, schedule, chunk, 0.5, None, p(conf_t), None, None, None, None, thr,
                                           p(hits_t), cap, p(n_hits), None)
    return rc, int(n_hits.item())


@gpu
def test_hits(fx):
    """The hit set is {q : conf[q] > t} of the per-window output, with capacity 0, a too small capacity (exact total, a
    subset of the hits) and hits-only calls; Python's re-run returns them all."""
    import torch
    models = [3, 2, 0, 5, 3, 11, 8, 1, 7]
    recs = [8, 8, 4, 8, 6, 5, 7, 8, 8]
    ref = _pairs(fx, models, recs, 'listener', 1024)
    for t in np.quantile(ref['conf'], [0.2, 0.6, 0.97]).tolist():
        want = np.nonzero(ref['conf'] > t)[0]
        assert 2 <= want.size < ref['conf'].size
        got = _pairs(fx, models, recs, 'listener', 1024, hit_threshold=t, hit_capacity=3)     # re-runs with room for all
        assert np.array_equal(got['hits'], want), t
        assert _same(got['conf'], ref['conf'])
        only = _pairs(fx, models, recs, 'listener', 1024, per_window=False, hit_threshold=t)
        assert np.array_equal(only['hits'], want) and _same(only['activations'], ref['activations'])
        rc, total = _raw_call(fx, models, recs, t, 0)                                          # count only
        assert rc == 0 and total == want.size
        cap = want.size // 2                                                                   # too small
        small = torch.full((cap + 1,), -1, dtype=torch.int64, device='cuda')
        rc, total = _raw_call(fx, models, recs, t, cap, small)
        h = small.cpu().numpy()
        assert rc == 0 and total == want.size and h[cap] == -1
        assert len(set(h[:cap])) == cap and set(h[:cap]) <= set(want.tolist())
        conf = torch.empty(ref['conf'].size, dtype=torch.float64, device='cuda')                # hits beside d_conf alone
        big = torch.empty(want.size + 3, dtype=torch.int64, device='cuda')
        rc, total = _raw_call(fx, models, recs, t, want.size + 3, big, conf)
        assert rc == 0 and total == want.size
        assert np.array_equal(np.sort(big[:total].cpu().numpy()), want) and _same(conf.cpu().numpy(), ref['conf'])


@gpu
def test_false_activations_pool(fx):
    """Equals false_activations on a two-model bank that holds the same network in slot 0, clips and indices alike, for
    pairs and for the cross product; calls regrouped by a small CORPUS_CALL_SAMPLES give the same outputs and hits."""
    from mycroft_precise_b200 import offline
    m = fx.m
    recs = fx.recs + [_noise(50000, 21)]
    for mid in (0, 2):
        model, pr, sens, lvl = fx.spec[mid]
        bank = m.PreciseB200(pr, hidden=model.hidden, activation=model.activation,
                             recurrent_activation=model.recurrent_activation)
        bank.load_weights(model.kernel, model.recurrent, model.bias, model.dense_w, model.dense_b)
        bank.add_model(fx.spec[1][0], fx.spec[1][1])
        cut = offline._chunk_cut(recs, 2048)
        conf = offline.score_corpus(bank, cut, 'listener', 2048, divisor=32767)['conf'][0].cpu().numpy()
        for t in np.quantile(conf, [0.5, 0.97]).tolist():
            want = offline.false_activations(bank, recs, 2048, t)
            assert want
            got = offline.false_activations_pool(fx.pool, recs, [mid], None, 2048, t)
            assert len(got) == len(want)
            for (p, r, k, clip), (i, kw, cw) in zip(got, want):
                assert (p, r, k) == (i, i, kw) and _same(clip, cw)
            rec_ids = [9, 8, 4, 9]
            got = offline.false_activations_pool(fx.pool, recs, [mid, 1, mid, mid], rec_ids, 2048, t)
            per_rec = {}
            for i, k, clip in want:
                per_rec.setdefault(i, []).append((k, clip))
            mine = [(r, k, clip) for p, r, k, clip in got if p != 1]
            expect = [(r, k, clip) for p, r in enumerate(rec_ids) if p != 1 for k, clip in per_rec.get(r, [])]
            assert [x[:2] for x in mine] == [x[:2] for x in expect]
            assert all(_same(a[2], b[2]) for a, b in zip(mine, expect))
        bank.close()


@gpu
def test_regrouped_calls(fx, monkeypatch):
    from mycroft_precise_b200 import offline
    recs = fx.recs + [_noise(50000, 21)]
    models = np.asarray([3, 2, 0, 5, 3, 11, 8, 1, 7, 4], np.int32)
    rec_ids = np.asarray([9, 8, 4, 8, 6, 5, 7, 0, 9, 1], np.int32)
    for schedule, chunk, hit in (('listener', 1024, 0.5), ('simulate', 4096, None)):
        one = offline.score_corpus_pairs(fx.pool, recs, models, rec_ids, schedule, chunk, hit_threshold=hit)
        with monkeypatch.context() as mp:
            mp.setattr(offline, 'CORPUS_CALL_SAMPLES', 30000)
            many = offline.score_corpus_pairs(fx.pool, recs, models, rec_ids, schedule, chunk, hit_threshold=hit)
            red = offline.score_corpus_pairs(fx.pool, recs, models, rec_ids, schedule, chunk, per_window=False,
                                             hit_threshold=hit)
        assert np.array_equal(one['pair_offsets'], many['pair_offsets'])
        for k in KEYS:
            if one[k] is None:
                assert many[k] is None
                continue
            assert _same(many[k].cpu().numpy(), one[k].cpu().numpy()), k
            if k not in WIN:
                assert _same(red[k].cpu().numpy(), one[k].cpu().numpy()), k
        if hit is not None:
            h = one['hits'].cpu().numpy()
            assert h.size and np.array_equal(many['hits'].cpu().numpy(), h) and np.array_equal(red['hits'].cpu().numpy(), h)
            assert np.array_equal(h, np.nonzero(one['conf'].cpu().numpy() > hit)[0])


@gpu
def test_simulate_pairs_matches_simulate_pool(fx):
    from mycroft_precise_b200 import offline
    recs = fx.recs + [_noise(40000, 9)]
    ids = np.asarray([1, 0, 2, 6, 10], np.int32)
    metrics, _ = offline.simulate_pool(fx.pool, recs, ids, 4096, 0.4)
    models = np.repeat(ids, len(recs))[::-1].copy()
    rec_ids = np.tile(np.arange(len(recs), dtype=np.int32), len(ids))[::-1].copy()
    got, totals = offline.simulate_pairs(fx.pool, recs, models, rec_ids, 4096, 0.4)
    row = {int(mid): i for i, mid in enumerate(ids)}
    for p, (mid, r) in enumerate(zip(models, rec_ids)):
        assert got[p] == metrics[row[int(mid)]][r], (p, mid, r)
    assert got[-1] is None                                          # recording 0 is empty
    assert sorted(totals) == sorted(row)
    for mid, t in totals.items():
        assert t.activations == sum(x.activations for x in metrics[row[mid]] if x is not None)
        assert t.seconds == sum(x.seconds for x in metrics[row[mid]][::-1] if x is not None)


@gpu
def test_oracle_anchor(fx):
    """Raw against the oracle listener on its own windows, and fired equals OracleTrigger replayed on the library's conf."""
    c = 1024
    models = [2, 0, 2]
    recs = [8, 4, 5]
    got = _pairs(fx, models, recs, 'listener', c)
    P = got['pair_offsets']
    worst = 0.0
    for p, (mid, r) in enumerate(zip(models, recs)):
        model, pr, sens, lvl = fx.spec[mid]
        sl = slice(P[p], P[p + 1])
        want = _oracle_listener(model, pr, fx.recs[r], c, sens, lvl)
        assert want.size == P[p + 1] - P[p]
        worst = max(worst, float(np.max(np.abs(got['raw'][sl] - want))))
        det = OracleTrigger(2 * c, sens, lvl)
        assert [bool(det.update(float(x))) for x in got['conf'][sl]] == list(got['fired'][sl].astype(bool)), p
    assert worst < 1e-5, worst
    assert got['fired'].sum() > 0


@gpu
def test_side_effects_and_refusals(fx):
    """Pair calls between pool ticks leave the ticks as a twin handle without them has them; a pool_load right after a
    queued call leaves that call's outputs the old model's; every refused call writes nothing and changes nothing."""
    import torch
    from mycroft_precise_b200.core import PBError
    m = fx.m
    S, K, chunk = 6, 6, 1024
    twins = []
    for _ in range(2):
        sb = m.StreamBatch(fx.spec[0][0], S, chunk_samples=chunk)
        sb.set_pool(len(fx.spec))
        for i, (model, pr, sens, lvl) in enumerate(fx.spec):
            sb.pool_load(i, model, pr, sensitivity=sens, trigger_level=lvl)
        sb.set_stream_pool(np.asarray([0, 2, 5, -1, 7, 2], np.int32))
        twins.append(sb)
    rs = np.random.RandomState(3)
    pcm = [torch.from_numpy(np.clip(rs.randn(S, chunk) * 3000, -32768, 32767).astype(np.int16)).cuda() for _ in range(K)]
    ref = fx.ref('listener', 1024)
    models, recs = np.asarray([3, 0, 3], np.int32), np.asarray([8, 4, 2], np.int32)
    outs = [[], []]
    for k in range(K):
        for t, sb in enumerate(twins):
            o = sb.update_pool(pcm[k])
            outs[t].append({x: o[x].cpu().numpy() for x in WIN})
            if t == 0:
                r = _host(sb.core.score_corpus_pairs(fx.pcm, fx.offsets, models, recs, 'listener', 1024))
                _check_pairs(r, ref, models, recs)
    for a, b in zip(*outs):
        for x in a:
            assert _same(a[x], b[x]), x
    assert np.array_equal(twins[0].core.stream_pool(), twins[1].core.stream_pool())
    core = twins[0].core
    res = core.score_corpus_pairs(fx.pcm, fx.offsets, models, recs, 'listener', 1024)
    core.pool_load(3, fx.spec[4][0], fx.spec[4][1], sensitivity=fx.spec[4][2], trigger_level=fx.spec[4][3])
    _check_pairs(_host(res), ref, models, recs)
    _check_pairs(_host(core.score_corpus_pairs(fx.pcm, fx.offsets, models, recs, 'listener', 1024)), ref,
                 [4, 0, 4], recs)
    for sb in twins:
        sb.core.close()

    lib, h = fx.pool.lib, fx.pool._h
    n = fx.n_rec
    act = torch.zeros(8, dtype=torch.int64, device='cuda')
    hits = torch.zeros(8, dtype=torch.int64, device='cuda')
    n_hits = torch.full((1,), -7, dtype=torch.int64, device='cuda')
    ok_m, ok_r = np.asarray([0, 1], np.int32), np.asarray([8, 4], np.int32)
    before = _pairs(fx, ok_m, ok_r, 'listener', 1024)
    p = lambda t: C.c_void_p(t.data_ptr())

    def call(models=ok_m, recs=ok_r, n_pairs=2, schedule=0, chunk=1024, divisor=32768, outs=True, cap=0, d_hits=None,
             d_n=None, above=None):
        pm = None if models is None else models.ctypes.data_as(C.c_void_p)
        pr = None if recs is None else recs.ctypes.data_as(C.c_void_p)
        return lib.pb_score_corpus_pairs(h, p(fx.pcm), fx.offsets.ctypes.data_as(C.c_void_p), n, pm, pr, n_pairs, divisor,
                                         schedule, chunk, 0.5, None, None, None, p(act) if outs else None, above, None,
                                         0.5, d_hits, cap, d_n, None)

    assert call(n_pairs=-1) == -1
    assert call(models=None) == -1 and call(recs=None) == -1
    assert call(models=np.asarray([0, 12], np.int32)) == -1                    # outside [0, max_models)
    assert call(models=np.asarray([-1, 0], np.int32)) == -1
    assert call(recs=np.asarray([0, n], np.int32)) == -1                       # outside [0, n_rec)
    assert call(recs=np.asarray([-1, 0], np.int32)) == -1
    assert call(outs=False) == -1                                              # every output null
    assert call(cap=-1, d_n=p(n_hits)) == -1
    assert call(cap=4, d_n=p(n_hits)) == -1                                    # null d_hits with a capacity
    assert call(cap=4, d_hits=p(hits)) == -1                                   # d_hits without d_n_hits
    assert call(schedule=1, chunk=4096, d_n=p(n_hits)) == -1                   # hits with the simulate schedule
    assert call(above=p(act)) == -1                                            # above with the listener schedule
    assert call(divisor=1000) == -1 and call(schedule=7) == -1
    assert call(schedule=1, chunk=10) == -1
    empty = m.PreciseB200()
    empty.set_pool(4)
    empty.pool_load(0, fx.spec[0][0])
    with pytest.raises(ValueError, match='holds no model'):
        empty.score_corpus_pairs(fx.pcm, fx.offsets, np.asarray([0, 1], np.int32), ok_r)
    empty.close()
    nopool = m.PreciseB200()
    with pytest.raises(PBError, match='no model pool'):
        nopool.score_corpus_pairs(fx.pcm, fx.offsets, ok_m, ok_r)
    nopool.close()
    assert not act.any() and not hits.any() and int(n_hits.item()) == -7      # refused calls wrote nothing
    assert call(n_pairs=0, d_n=p(n_hits)) == 0 and int(n_hits.item()) == 0     # nothing to score: no hits
    after = _pairs(fx, ok_m, ok_r, 'listener', 1024)
    for k in KEYS:
        assert (before[k] is None and after[k] is None) or _same(before[k], after[k]), k


def test_null_handle_without_gpu():
    """The new entry points refuse a null handle before touching the device."""
    import __graft_entry__ as g
    from mycroft_precise_b200.core import lib_path
    if not os.path.isfile(lib_path()):
        g.build()
    from mycroft_precise_b200.core import get_lib
    lib = get_lib()
    offs = np.asarray([0, 0], np.int64)
    ids = np.zeros(1, np.int32)
    assert lib.pb_score_corpus_pairs(None, None, offs.ctypes.data_as(C.c_void_p), 1, ids.ctypes.data_as(C.c_void_p),
                                     ids.ctypes.data_as(C.c_void_p), 1, 32768, 0, 1024, 0.5, None, None, None, None, None,
                                     None, 0.5, None, 0, None, None) == -1
    assert b'null handle' in lib.pb_last_error()
    assert lib.pb_debug_corpus_pairs_batch(None, 0) == -1
