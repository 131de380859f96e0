"""Pool models over labelled clips (pb_score_dataset, PreciseB200.score_dataset, offline.test_pool / calc_threshold,
StreamBatch.pool_calibrate).  The window is checked against pb_score_corpus_pool (bit for bit, where the two schedules
coincide) and against the float64 oracle's vectorize; the statistics against their numpy restatement (oracle/dataset.py) on the
call's own outputs.  -m gpu."""
import ctypes as C

import numpy as np
import pytest

from oracle import dataset as od
from oracle import gru as og
from oracle import mfcc as om
from oracle.params import OracleParams

gpu = pytest.mark.gpu
MAX = 24000                                   # ListenerParams().max_samples


def _mod():
    import mycroft_precise_b200 as m
    return m


def _noise(n, seed, sigma=3000):
    rs = np.random.RandomState(seed)
    return np.clip(rs.randn(n) * sigma * (1 + np.sin(np.arange(n) / 4000.0)), -32768, 32767).astype(np.int16)


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def _models(m):
    """Twelve fused networks, H = 8 .. 24, every third with tanh / sigmoid activations; dense biases spread the outputs over
    (0, 1).  Slots 12 and 13 saturate: they output exactly 1.0 and exactly 0.0."""
    out = []
    for i in range(12):
        g = m.GruModel.random(13, [20, 12, 24, 16, 8][i % 5], seed=200 + i, scale=0.1)
        if i % 3 == 2:
            g.activation, g.recurrent_activation = 'tanh', 'sigmoid'
        g.dense_b = 1.5 - 0.5 * (i % 7)
        out.append(g)
    for b in (100.0, -100.0):
        g = m.GruModel.random(13, 20, seed=300, scale=0.01)
        g.dense_b = b
        out.append(g)
    return out


def _pack(clips, lead=0):
    """Clips back to back after ``lead`` samples of another clip (so offsets need not be multiples of 8)."""
    parts = ([_noise(lead, 999)] if lead else []) + list(clips)
    offsets = np.concatenate([[0], np.cumsum([len(c) for c in parts])]).astype(np.int64)
    return np.concatenate(parts), offsets


class Fixture:
    def __init__(self):
        import torch
        m = _mod()
        self.m, self.torch = m, torch
        self.models = _models(m)
        self.core = m.PreciseB200()
        self.core.set_pool(len(self.models) + 2)              # the last two slots stay empty
        for i, g in enumerate(self.models):
            self.core.pool_load(i, g)
        rs = np.random.RandomState(5)
        lens = [1, 511, 1599, 1600, 2400, 24000, 24001, 30001] + rs.randint(800, 40000, 292).tolist()
        self.clips = [_noise(n, 1000 + i) for i, n in enumerate(lens)]
        self.targets = (rs.rand(len(lens)) < 0.4).astype(np.uint8)
        pcm, self.offsets = _pack(self.clips)
        self.pcm = torch.from_numpy(pcm).cuda()
        self.n = len(lens)
        self.ids = np.arange(12, dtype=np.int32)

    def dev(self, a):
        return self.torch.from_numpy(a).cuda()

    def close(self):
        self.core.close()


@pytest.fixture(scope='module')
def fx():
    pytest.importorskip('torch')
    f = Fixture()
    yield f
    f.close()


def _host(res):
    return {k: (v.cpu().numpy() if hasattr(v, 'cpu') else v) for k, v in res.items() if v is not None}


def _check_stats(res, raw, targets, thr, rows=None, k=None):
    """count / hist / fit of a call against the numpy restatement on raw ([k, n], or [n_pairs] with rows)."""
    thr = np.asarray(thr, np.float32)
    k = raw.shape[0] if rows is None else k
    for i in range(k):
        x, t = (raw[i], targets) if rows is None else (raw[rows == i], targets[rows == i])
        count, hist, fit = od.dataset_stats(x, t, thr)
        assert np.array_equal(res['count'][i], count), i
        assert np.array_equal(res['hist'][i], hist), i
        assert np.array_equal(res['fit'][i][:, 0], fit[:, 0]), i
        assert np.all(np.abs(res['fit'][i][:, 1:] - fit[:, 1:]) <= fit[:, :1]), (i, res['fit'][i], fit)


# ---- 1. the window ---------------------------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize('L', [1, 511, 1599, 1600, 24000])
def test_short_clip_is_listener_window_0(fx, L):
    """L <= max_samples: the same frames, start row and scan as the listener schedule's first window with chunk = L."""
    clip = _noise(L, 40 + L)
    pcm, offsets = fx.dev(clip), np.asarray([0, L], np.int64)
    want = fx.core.score_corpus_pool(pcm, offsets, fx.ids, 'listener', L, divisor=32767)['raw'].cpu().numpy()
    got = fx.core.score_dataset(pcm, offsets, np.ones(1, np.uint8), fx.ids)['raw'].cpu().numpy()
    assert want.shape == (12, 1) and _same(got, want)
    if L < 1600:                                              # no frame: the all-zero input
        zero = fx.core.score_dataset(fx.dev(np.zeros(5, np.int16)), np.asarray([0, 5], np.int64), np.ones(1, np.uint8), fx.ids)
        assert _same(got, zero['raw'].cpu().numpy())


@gpu
def test_long_clips_are_cropped_to_their_last_samples(fx):
    """Longer than max_samples, with an excess that is not a multiple of the hop or of 8, at odd packed offsets: the float64
    oracle's vectorize, and bit for bit the same call on the clips cropped beforehand."""
    lens = [MAX + 1, MAX + 7, MAX + 800, MAX + 12345, 100000, 24001, 1600, 511]
    clips = [_noise(n, 70 + i) for i, n in enumerate(lens)]
    pcm, offsets = _pack(clips, lead=3)
    tg = np.ones(len(offsets) - 1, np.uint8)
    ids = np.asarray([0, 2, 4], np.int32)
    got = fx.core.score_dataset(fx.dev(pcm), offsets, tg, ids)['raw'].cpu().numpy()[:, 1:]
    opr = OracleParams()
    worst = 0.0
    for row, mid in enumerate(ids):
        g = fx.models[mid]
        w = og.GruWeights(g.kernel, g.recurrent, g.bias, g.dense_w, g.dense_b, activation=g.activation,
                          recurrent_activation=g.recurrent_activation)
        for j, c in enumerate(clips):
            feats = om.vectorize(c.astype(np.float64) / 32767.0, opr)
            want = og.gru_forward(w, feats[None], dtype=np.float64)[0][0]
            worst = max(worst, abs(float(got[row, j]) - float(want)))
    assert worst < 1e-5, worst
    fx.core.force_generic(True)
    try:
        a = fx.core.score_dataset(fx.dev(pcm), offsets, tg, ids)['raw'].cpu().numpy()[:, 1:]
        cpcm, coff = _pack([c[-MAX:] for c in clips], lead=5)
        b = fx.core.score_dataset(fx.dev(cpcm), coff, tg, ids)['raw'].cpu().numpy()[:, 1:]
    finally:
        fx.core.force_generic(False)
    assert _same(a, b)
    assert np.max(np.abs(a - got)) < 1e-5                     # the fast and the generic K1 agree to the same bar


# ---- 2. statistics -----------------------------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize('n_thr', [1, 100, 1024])
def test_statistics_equal_numpy_on_the_calls_raw(fx, n_thr):
    ids = np.arange(14, dtype=np.int32)                        # with the two saturated networks
    raw = fx.core.score_dataset(fx.pcm, fx.offsets, fx.targets, ids)['raw'].cpu().numpy()
    assert (raw[12] == 1.0).all() and (raw[13] == 0.0).all() and 0.05 < (raw[:12] > 0.5).mean() < 0.95
    if n_thr == 1:
        thr = np.float32([0.5])
    else:                                                      # eight thresholds that equal outputs, the rest a grid
        hits = np.unique(raw[:12].ravel()[::90])[::5][:8]
        grid = np.setdiff1d(np.linspace(0.001, 0.999, 2 * n_thr).astype(np.float32), hits)
        thr = np.sort(np.concatenate([hits, grid[::2][:n_thr - len(hits)]]))
    assert len(thr) == n_thr and np.all(np.diff(thr) > 0)
    res = _host(fx.core.score_dataset(fx.pcm, fx.offsets, fx.targets, ids, thresholds=thr))
    assert _same(res['raw'], raw) and _same(res['thresholds'], thr)
    _check_stats(res, raw, fx.targets, thr)
    assert res['fit'][12].sum() == 0 and res['fit'][13].sum() == 0 and res['fit'][:12, :, 0].sum() == 12 * fx.n
    if n_thr > 1:
        assert res['hist'][:12, :, 1::2].sum() >= 8            # outputs equal to a threshold were met
    # DatasetStats on the device's numbers = the reference's comparisons on the outputs
    from mycroft_precise_b200.offline import DatasetStats, calc_threshold
    st = DatasetStats(thr, res['count'][3], res['hist'][3], res['fit'][3])
    pos = fx.targets != 0
    for t in thr[:: max(1, len(thr) // 7)]:
        assert st.false_pos(t) == int((raw[3][~pos] > t).sum()) and st.false_neg(t) == int((~(raw[3][pos] > t)).sum())
        assert st.num_correct(t) == int(((raw[3] >= t) == pos).sum())
    mu, std = calc_threshold(st)
    o_mu, o_std = od.calc_threshold(raw[3], fx.targets)
    assert abs(mu - o_mu) < 1e-4 and abs(std - o_std) < 1e-4


# ---- 3. shapes ---------------------------------------------------------------------------------------------------------------

THR = [0.1, 0.5, 0.9]


@gpu
def test_cross_product_equals_pairs(fx):
    ids = np.asarray([3, 2, 3, 11, 0, 8], np.int32)            # repeated ids, both activation classes
    cross = _host(fx.core.score_dataset(fx.pcm, fx.offsets, fx.targets, ids, thresholds=THR, miss_threshold=0.5))
    assert _same(cross['raw'][0], cross['raw'][2]) and np.array_equal(cross['hist'][0], cross['hist'][2])
    rows = np.repeat(np.arange(len(ids)), fx.n).astype(np.int32)
    recs = np.tile(np.arange(fx.n), len(ids)).astype(np.int32)
    pairs = _host(fx.core.score_dataset(fx.pcm, fx.offsets, fx.targets, ids, rows, recs, thresholds=THR, miss_threshold=0.5))
    assert _same(pairs['raw'], cross['raw'].ravel())
    for key in ('count', 'hist', 'fit', 'misses'):
        assert np.array_equal(pairs[key], cross[key]), key
    # any order, partial tiles, rows that score nothing
    rs = np.random.RandomState(3)
    sel = rs.permutation(len(rows))[:700]
    sel = sel[rows[sel] != 4]
    got = _host(fx.core.score_dataset(fx.pcm, fx.offsets, fx.targets, ids, rows[sel], recs[sel], thresholds=THR))
    assert _same(got['raw'], cross['raw'].ravel()[sel]) and got['count'][4].sum() == 0
    _check_stats(got, got['raw'], fx.targets[recs[sel]], THR, rows=rows[sel], k=len(ids))


@gpu
def test_batches_with_and_without_raw(fx):
    ids = np.arange(12, dtype=np.int32)
    whole = _host(fx.core.score_dataset(fx.pcm, fx.offsets, fx.targets, ids, thresholds=THR, miss_threshold=0.5))
    rows = np.repeat(np.arange(12), 50).astype(np.int32)
    recs = np.tile(np.arange(50) * 5, 12).astype(np.int32)
    pwhole = _host(fx.core.score_dataset(fx.pcm, fx.offsets, fx.targets, ids, rows, recs, thresholds=THR, miss_threshold=0.5))
    fx.core.corpus_pool_rows(5)
    fx.core.corpus_pairs_batch(97)
    try:
        for per_entry in (True, False):
            got = _host(fx.core.score_dataset(fx.pcm, fx.offsets, fx.targets, ids, thresholds=THR, per_entry=per_entry,
                                              miss_threshold=0.5))
            pgot = _host(fx.core.score_dataset(fx.pcm, fx.offsets, fx.targets, ids, rows, recs, thresholds=THR,
                                               per_entry=per_entry, miss_threshold=0.5))
            assert ('raw' in got) == per_entry and ('raw' in pgot) == per_entry
            for ref, res in ((whole, got), (pwhole, pgot)):
                for key in res:
                    assert _same(np.asarray(res[key]), np.asarray(ref[key])), (per_entry, key)
    finally:
        fx.core.corpus_pool_rows(0)
        fx.core.corpus_pairs_batch(0)


@pytest.fixture
def generic_k1(fx):
    yield
    fx.core.force_generic(False)


@gpu
def test_two_calls_add_up_and_test_pool_splits(fx, monkeypatch, generic_k1):
    from mycroft_precise_b200 import offline
    ids = np.asarray([1, 5, 9], np.int32)
    # one K1 kernel for every clip wherever it is packed, so that raw is the same bit for bit in every call below
    fx.core.force_generic(True)
    whole = _host(fx.core.score_dataset(fx.pcm, fx.offsets, fx.targets, ids, thresholds=THR))
    h = fx.n // 2
    parts = []
    for sl in (slice(0, h), slice(h, None)):
        pcm, off = _pack(fx.clips[sl], lead=1)
        tg = np.concatenate([[0], fx.targets[sl]]).astype(np.uint8)
        rows = np.repeat(np.arange(3), len(tg) - 1).astype(np.int32)
        recs = np.tile(np.arange(1, len(tg)), 3).astype(np.int32)     # every clip but the lead
        parts.append(_host(fx.core.score_dataset(fx.dev(pcm), off, tg, ids, rows, recs, thresholds=THR, per_entry=False)))
    for key in ('count', 'hist', 'fit'):
        assert np.array_equal(parts[0][key] + parts[1][key], whole[key]), key
    # offline.test_pool over several library calls, cross product and pairs, with the misclassified clips
    monkeypatch.setattr(offline, 'CORPUS_CALL_SAMPLES', 1 << 20)
    assert len(offline._call_groups(fx.clips)) > 3
    stats, missed = offline.test_pool(fx.core, fx.clips, fx.targets, ids, thresholds=THR, misses=True)
    raw = whole['raw']
    pos = fx.targets != 0
    for i in range(3):
        for key in ('count', 'hist', 'fit'):
            assert np.array_equal(getattr(stats[i], key), whole[key][i]), (i, key)
        assert np.array_equal(missed[i], np.nonzero((raw[i] > np.float32(0.5)) != pos)[0]) and len(missed[i]) > 0
    own = np.arange(fx.n) % 3
    ps = offline.test_pool(fx.core, fx.clips, fx.targets, ids, rows=own, recs=np.arange(fx.n), thresholds=THR)
    for i in range(3):
        assert np.array_equal(ps[i].count, np.bincount(fx.targets[own == i], minlength=2))
        assert len(ps[i]) == int((own == i).sum())
        assert np.array_equal(ps[i].hist, od.dataset_stats(raw[i][own == i], fx.targets[own == i], THR)[1])


# ---- 4. misses ---------------------------------------------------------------------------------------------------------------

@gpu
def test_misses_exact_set_capacity_and_rerun(fx):
    torch = fx.torch
    ids = np.asarray([0, 7], np.int32)
    res = _host(fx.core.score_dataset(fx.pcm, fx.offsets, fx.targets, ids, miss_threshold=0.6))
    want = np.nonzero(((res['raw'] > np.float32(0.6)) != (fx.targets != 0)[None]).ravel())[0]
    assert len(want) > 20 and np.array_equal(res['misses'], want)
    small = _host(fx.core.score_dataset(fx.pcm, fx.offsets, fx.targets, ids, miss_threshold=0.6, miss_capacity=3))
    assert np.array_equal(small['misses'], want)               # the second run with room for all of them
    none = _host(fx.core.score_dataset(fx.pcm, fx.offsets, fx.targets, ids, miss_threshold=0.6, miss_capacity=0))
    assert np.array_equal(none['misses'], want)
    # the C call itself: the count runs past the capacity, the list holds that many of the set
    n_miss = torch.zeros(1, dtype=torch.int64, device='cuda')
    d_miss = torch.full((8,), -1, dtype=torch.int64, device='cuda')
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = fx.core.lib.pb_score_dataset(fx.core._h, fx.pcm.data_ptr(), vp(fx.offsets), fx.n, vp(fx.targets), vp(ids), 2, None, None,
                                      0, 32767, MAX, None, 0, None, None, None, None, 0.6, d_miss.data_ptr(), 5,
                                      n_miss.data_ptr(), None)
    assert rc == 0
    torch.cuda.synchronize()
    got = d_miss.cpu().numpy()
    assert int(n_miss.item()) == len(want) and (got[5:] == -1).all() and len(set(got[:5])) == 5 and set(got[:5]) <= set(want)


# ---- 5. contract -------------------------------------------------------------------------------------------------------------

@gpu
def test_refused_calls(fx):
    m, core, lib = fx.m, fx.core, fx.core.lib
    torch = fx.torch
    vp = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
    ids = np.asarray([0, 1], np.int32)
    count = torch.full((2, 2), 7, dtype=torch.int64, device='cuda')
    raw = torch.zeros((2, fx.n), dtype=torch.float32, device='cuda')
    thr = np.asarray([0.25, 0.5])
    rows, recs = np.asarray([0, 1], np.int32), np.asarray([0, 1], np.int32)

    def call(h=None, pcm=fx.pcm.data_ptr(), offsets=fx.offsets, n_rec=fx.n, targets=fx.targets, ids=ids, k=2, rows=None,
             recs=None, n_pairs=0, divisor=32767, max_samples=MAX, thr=thr, n_thr=2, raw=raw.data_ptr(),
             count=count.data_ptr(), hist=None, fit=None, miss=None, cap=0, n_miss=None):
        return lib.pb_score_dataset(core._h if h is None else h, pcm, vp(offsets), n_rec, vp(targets), vp(ids), k, vp(rows),
                                    vp(recs), n_pairs, divisor, max_samples, vp(thr), n_thr, raw, count, hist, fit, 0.5, miss,
                                    cap, n_miss, None)

    assert call() == 0
    hist = torch.zeros((2, 2, 5), dtype=torch.int64, device='cuda')
    fit = torch.zeros((2, 2, 3), dtype=torch.int64, device='cuda')
    empty = fx.offsets.copy()
    empty[4] = empty[5]
    bad = [dict(pcm=None), dict(offsets=None), dict(n_rec=-1), dict(targets=None), dict(ids=None), dict(k=-1),
           dict(ids=np.asarray([0, 14], np.int32)), dict(ids=np.asarray([0, 99], np.int32)), dict(ids=np.asarray([-1, 0], np.int32)),
           dict(rows=rows, n_pairs=2), dict(recs=recs, n_pairs=2), dict(n_pairs=-1),
           dict(rows=np.asarray([0, 2], np.int32), recs=recs, n_pairs=2), dict(rows=rows, recs=np.asarray([0, fx.n], np.int32), n_pairs=2),
           dict(rows=rows, recs=np.asarray([-1, 0], np.int32), n_pairs=2),
           dict(divisor=1000), dict(max_samples=0), dict(offsets=empty), dict(offsets=fx.offsets[::-1].copy()),
           dict(n_thr=1025), dict(n_thr=-1), dict(thr=None), dict(thr=np.asarray([0.5, 0.5])), dict(thr=np.asarray([0.5, 0.25])),
           dict(thr=np.asarray([0.5, 0.5 + 1e-12])), dict(thr=np.asarray([np.nan, 0.5])),
           dict(hist=hist.data_ptr(), n_thr=0), dict(raw=None, count=None), dict(cap=-1, n_miss=count.data_ptr()),
           dict(cap=4, n_miss=count.data_ptr()), dict(miss=count.data_ptr())]
    for kw in bad:
        assert call(**kw) == -1, kw
        assert lib.pb_last_error()
    assert lib.pb_score_dataset(None, None, None, 0, None, None, 0, None, None, 0, 32767, MAX, None, 0, None, None, None, None,
                                0.5, None, 0, None, None) == -1
    torch.cuda.synchronize()
    assert not (count == 7).any()                               # only the accepted call wrote
    # the fit's sums hold 2^24 entries of one (row, label): refused before anything runs, and only with d_fit
    n_big = (1 << 24) + 1
    big_off = np.arange(n_big + 1, dtype=np.int64)
    big_pcm = torch.zeros(n_big, dtype=torch.int16, device='cuda')
    big_t = np.zeros(n_big, np.uint8)
    assert call(pcm=big_pcm.data_ptr(), offsets=big_off, n_rec=n_big, targets=big_t, raw=None, fit=fit.data_ptr()) == -1
    assert b'2^24' in lib.pb_last_error()
    # no pool
    plain = m.PreciseB200()
    try:
        assert call(h=plain._h) == -4
        with pytest.raises(m.PBError):
            plain.score_dataset(fx.pcm, fx.offsets, fx.targets, ids)
    finally:
        plain.close()
    with pytest.raises(ValueError):
        core.score_dataset(fx.pcm, fx.offsets, fx.targets, ids, rows=rows)
    with pytest.raises(ValueError):
        core.score_dataset(fx.pcm, fx.offsets, fx.targets.astype(np.int32), ids)
    # no entry at all: zeroed statistics, nothing scored
    for res in (core.score_dataset(fx.pcm, fx.offsets, fx.targets, ids[:0]),
                core.score_dataset(fx.pcm, fx.offsets, fx.targets, ids, rows[:0], recs[:0], miss_threshold=0.5)):
        assert int(res['count'].sum()) == 0 and int(res['hist'].sum()) == 0 and res['raw'].numel() == 0


@gpu
def test_scoring_a_dataset_leaves_the_streams_alone(fx):
    import torch
    m = fx.m
    S, chunk, K = 8, 1024, 10
    audio = np.stack([_noise(K * chunk, 500 + s) for s in range(S)])

    def run(score):
        sb = m.StreamBatch(fx.models[0], S, chunk_samples=chunk)
        sb.set_pool(4)
        for i in range(4):
            sb.pool_load(i, fx.models[i])
        sb.set_stream_pool(np.asarray([0, 1, 2, 3, 0, 1, -1, 2], np.int32))
        outs = []
        for k in range(K):
            if score and k == K // 2:
                sb.core.score_dataset(fx.pcm, fx.offsets, fx.targets, np.asarray([1, 3], np.int32), thresholds=THR,
                                      miss_threshold=0.5)
            o = sb.update_all(torch.from_numpy(audio[:, k * chunk:(k + 1) * chunk].copy()).cuda())
            outs.append({key: o[key].cpu().numpy().copy() for key in ('raw', 'conf', 'fired')})
        pool = sb.stream_pool()
        sb.core.close()
        return outs, pool

    a, pa = run(False)
    b, pb = run(True)
    assert np.array_equal(pa, pb)
    for x, y in zip(a, b):
        for key in x:
            assert _same(x[key], y[key]), key


@gpu
def test_pool_calibrate(fx):
    import torch
    m = fx.m
    S, chunk = 4, 1024
    clips = fx.clips[8:60]
    sb = m.StreamBatch(fx.models[0], S, chunk_samples=chunk)
    sb.set_pool(3)
    for i in range(3):
        sb.pool_load(i, fx.models[i + 1], sensitivity=0.6, trigger_level=2)
    sb.set_stream_pool(np.asarray([0, 1, 2, 1], np.int32))
    pcm = torch.from_numpy(np.stack([_noise(chunk * 30, 600 + s) for s in range(S)])).cuda()
    before = [sb.update_pool(pcm[:, k * chunk:(k + 1) * chunk].contiguous())['conf'].cpu().numpy().copy() for k in range(30)]
    ids = np.asarray([0, 2], np.int32)
    rows = (np.arange(len(clips)) % 2).astype(np.int32)
    fits = sb.pool_calibrate(ids, clips, rows, np.arange(len(clips)))
    # the fit: calc_threshold's expression on each model's own clips
    for j, mid in enumerate(ids):
        own = [c for c, r in zip(clips, rows) if r == j]
        p, off = _pack(own)
        raw = sb.core.score_dataset(torch.from_numpy(p).cuda(), off, np.ones(len(own), np.uint8), ids[j:j + 1])['raw'].cpu().numpy()[0]
        mu, std = od.calc_threshold(raw, np.ones(len(own)))
        assert abs(fits[j][0] - mu) < 1e-4 and abs(fits[j][1] - std) < 1e-4 and std > 0
    # a freshly loaded pool with the fitted threshold_config gives the same conf on the same ticks
    ref = m.StreamBatch(fx.models[0], S, chunk_samples=chunk)
    ref.set_pool(3)
    for i in range(3):
        pr = m.ListenerParams(threshold_config=(fits[[0, None, 1][i]],)) if i != 1 else None
        ref.pool_load(i, fx.models[i + 1], pr, sensitivity=0.6, trigger_level=2)
    ref.set_stream_pool(np.asarray([0, 1, 2, 1], np.int32))
    sb.clear()
    changed = False
    for k in range(30):
        tick = pcm[:, k * chunk:(k + 1) * chunk].contiguous()
        a, b = sb.update_pool(tick), ref.update_pool(tick)
        for key in ('raw', 'conf', 'fired'):
            assert _same(a[key].cpu().numpy(), b[key].cpu().numpy()), (k, key)
        conf = a['conf'].cpu().numpy()
        changed |= bool((conf[[0, 2]] != before[k][[0, 2]]).any())
        assert _same(conf[[1, 3]], before[k][[1, 3]])            # slot 1 was not calibrated
    assert changed
    sb.core.close()
    ref.core.close()


@gpu
def test_command_line(fx, tmp_path, capsys):
    """python -m mycroft_precise_b200.test with two models: per model a heading, the misclassified files, precise-test's
    two blocks and the calc-threshold line, all as numpy gives them from the same clips' outputs."""
    import wave
    from mycroft_precise_b200 import test as cli
    idx = list(range(4, 44))
    names = {}
    for i in idx:
        d = tmp_path / 'data' / 'test' / ('wake-word' if fx.targets[i] else 'not-wake-word')
        d.mkdir(parents=True, exist_ok=True)
        names[i] = str(d / ('clip%03d.wav' % i))
        with wave.open(names[i], 'wb') as w:
            w.setnchannels(1); w.setsampwidth(2); w.setframerate(16000); w.writeframes(fx.clips[i].tobytes())
    paths = []
    for j in (1, 2):
        paths.append(str(tmp_path / ('model%d.npz' % j)))
        fx.m.save_weights(paths[-1], fx.models[j])
    cli.main(paths + [str(tmp_path / 'data'), '-t', '0.4', '--calc-threshold'])
    out = ''.join(l for l in capsys.readouterr().out.splitlines(True) if not l.startswith('Warning:'))
    pcm, off = _pack([fx.clips[i] for i in idx])
    tg = fx.targets[idx]
    raw = fx.core.score_dataset(fx.dev(pcm), off, tg, np.asarray([1, 2], np.int32))['raw'].cpu().numpy()
    blocks = out.split('=== %s ===\n' % paths[1])
    assert len(blocks) == 2 and blocks[0].startswith('=== %s ===\n' % paths[0])
    for row, text in enumerate(blocks):
        x, pos = raw[row], tg != 0
        act = x > np.float32(0.4)
        fp = {names[i] for i, a, p in zip(idx, act, pos) if a and not p}
        fn = {names[i] for i, a, p in zip(idx, act, pos) if not a and p}
        head, rest = text.split('=== False Negatives ===\n')
        assert set(head.split('=== False Positives ===\n')[1].split()) == fp
        assert set(rest.split('=== Counts ===')[0].split()) == fn
        correct = int(((x >= np.float32(0.4)) == pos).sum())
        want = ('=== Counts ===\nFalse Positives: %d\nTrue Negatives: %d\nFalse Negatives: %d\nTrue Positives: %d\n\n\n'
                '=== Summary ===\n%d out of %d\n%s\n\n%s false positives\n%s false negatives\n\n'
                % (len(fp), int((~pos).sum()) - len(fp), len(fn), int(pos.sum()) - len(fn), correct, len(idx),
                   '{:.2%}'.format(correct / len(idx)), '{:.2%}'.format(len(fp) / max(1, int((~pos).sum()))),
                   '{:.2%}'.format(len(fn) / max(1, int(pos.sum())))))
        assert want in text
        mu, std = od.calc_threshold(x, tg)
        assert text.rstrip().endswith('Peak: {:.2f} mu, {:.2f} std'.format(mu, std))
