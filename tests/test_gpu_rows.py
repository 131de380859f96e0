"""Networks given as weight rows over labelled network inputs (pb_score_rows; PreciseB200.score_rows, offline.test_rows and the
test command's path for networks of more than 24 units).

1. Raw bit for bit against pb_predict on a handle holding each network (gru_wide_kernel): H 1 .. 128 over every HP / 16 and
   partial last warps, the four activation pairs in rotation, both strides where H <= 24, n = 1, 127, 128, 129, 300 and 10 000.
2. The default shape (H 20, F 13, linear / hard_sigmoid, which pb_predict scores on its own kernels) and every front end
   pb_vectorize_clips accepts, against float64 with test_gpu_wide_scan's gru_wide_kernel rule.
3. Independence of the other rows, their order and the groups and batches the call is cut into.
4. Statistics against numpy on the call's raw (test_gpu_dataset's check), without raw, added over calls cut at a multiple of
   16 clips, and pairs (random clips, networks interleaved, cut anywhere) bit-identical to the cross product's entries.
5. From training: the chirp task at H = 64 and a fused TrainState.
6. Refusals write nothing; stream state, pool and detectors are untouched.
7. The test command on a folder with 20-, 64- and 128-unit networks.

-m gpu throughout."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_dataset as td  # noqa: E402
import test_gpu_train_sweep as sw  # noqa: E402
import test_gpu_train_wide as tw  # noqa: E402
import test_gpu_wide_scan as ws  # noqa: E402
import train_task  # noqa: E402

gpu = pytest.mark.gpu
ACTS = (('linear', 'hard_sigmoid'), ('tanh', 'sigmoid'), ('linear', 'sigmoid'), ('tanh', 'hard_sigmoid'))
HIDDEN = (1, 7, 17, 24, 25, 31, 32, 33, 48, 63, 64, 65, 81, 96, 100, 112, 113, 127, 128)
SIZES = (1, 127, 128, 129, 300)
TS, WS = 2980, 55812


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def _clips(n, seed=0):
    """Noise, silence and chirp clips in turn (train_task's clips, lengths 12 000 .. 20 000)."""
    out = []
    for i in range(n):
        kind = i % 3
        c = train_task.clip(seed + i, kind == 2)
        out.append(np.zeros_like(c) if kind == 1 else c)
    return out


def _model(m, F, H, act, seed, family='std'):
    g = ws.FAMILIES[family](F, H, seed, act)
    return m.GruModel(g.kernel.astype(np.float32), g.recurrent.astype(np.float32), g.bias.astype(np.float32),
                      g.dense_w.astype(np.float32), np.float32(g.dense_b), act[0], act[1])


def _state(m, core, models, stride):
    """A TrainState of ``models`` at the given stride (from_models picks the wide one only past 24 units)."""
    import torch
    st = m.offline.TrainState.from_models(core, models, list(range(len(models))))
    if st.stride != stride:
        w = np.zeros((len(models), stride), np.float32)
        n = min(stride, st.stride)
        w[:, :n] = st.weights.cpu().numpy()[:, :n]
        st = m.offline.TrainState(core, torch.from_numpy(w).cuda(), torch.zeros((len(models), stride), device='cuda'),
                                  st.hidden, st.activation, st.recurrent_activation, st.seeds)
    return st


def _predict(m, pr, g, x):
    h = m.PreciseB200(pr, hidden=g.hidden, activation=g.activation, recurrent_activation=g.recurrent_activation)
    h.load_weights(g.kernel, g.recurrent, g.bias, g.dense_w, g.dense_b)
    out = h.predict(x).cpu().numpy().reshape(-1)
    h.close()
    return out


@pytest.fixture(scope='module')
def fx():
    pytest.importorskip('torch')
    f = sw.Fixture()
    core = f.core('default')
    f.x = f.m.offline.vectorize_clips(core, _clips(300))
    f.tg = (np.arange(300) % 3 == 2).astype(np.uint8)
    yield f
    f.close()


def _raw(core, st, x, tg, **kw):
    return core.score_rows(x, tg, st.rows, st.weights, **kw)['raw'].cpu().numpy()


# ---- 1. bit for bit against pb_predict ------------------------------------------------------------------------------------------

@gpu
def test_raw_is_pb_predict_bit_for_bit(fx):
    m, torch = fx.m, fx.torch
    core = fx.core('default')
    pr = m.ListenerParams()
    F = core.feature_size
    models = [_model(m, F, H, ACTS[i % 4], 100 + i) for i, H in enumerate(HIDDEN)]
    fused = [g for g in models if g.hidden <= 24]
    big = fx.x[torch.from_numpy(np.random.RandomState(1).randint(0, 300, 10000)).cuda()].contiguous()
    wide_st, fused_st = _state(m, core, models, WS), _state(m, core, fused, TS)
    for x in [fx.x[:n].contiguous() for n in SIZES] + [big]:
        n = x.shape[0]
        tg = np.zeros(n, np.uint8)
        got_w, got_f = _raw(core, wide_st, x, tg), _raw(core, fused_st, x, tg)
        for i, g in enumerate(models):
            want = _predict(m, pr, g, x)
            assert _same(got_w[i], want), (n, g.hidden, g.activation, g.recurrent_activation)
            if g.hidden <= 24:
                assert _same(got_f[fused.index(g)], want), (n, g.hidden, 'fused stride')


# ---- 2. float64 anchor ----------------------------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize('front', ['default', 'f1', 'f5', 'f16', 'mels16', 't1', 't73', 't112'])
def test_against_float64(fx, front):
    m = fx.m
    core = fx.core(front)
    F, T = core.feature_size, core.n_features
    x = m.offline.vectorize_clips(core, _clips(120, 7))
    xh = x.cpu().numpy()
    stats = {}
    for fam in ('std', 'keras 1', 'keras 1.3'):
        g = _model(m, F, 20, ACTS[0], 3, fam)
        st = _state(m, core, [g], TS)
        raw = _raw(core, st, x, np.zeros(x.shape[0], np.uint8))[0]
        ws.check(raw, None, ws.refs(ws.weights(g), xh, 'wide'), 'wide', g, T, '%s %s' % (front, fam), stats)
    print('rows float64 %s:' % front, {k: v for k, v in stats.items() if not k.startswith('_')})


# ---- 3. independence ------------------------------------------------------------------------------------------------------------

@gpu
def test_rows_do_not_depend_on_each_other_or_the_cut(fx):
    m = fx.m
    core = fx.core('default')
    F = core.feature_size
    rs = np.random.RandomState(4)
    models = [_model(m, F, int(rs.choice(HIDDEN)), ACTS[i % 4], 300 + i) for i in range(80)]
    order = rs.permutation(80)
    x, tg = fx.x[:129].contiguous(), fx.tg[:129]
    st = _state(m, core, [models[i] for i in order], WS)
    core.rows_groups(7, 3 * 129)
    try:
        cut = _raw(core, st, x, tg)
        pairs = core.score_rows(x, tg, st.rows, st.weights, np.repeat(np.arange(80), 129).astype(np.int32),
                                np.tile(np.arange(129), 80).astype(np.int32))['raw'].cpu().numpy()
    finally:
        core.rows_groups(0, 0)
    for j, i in enumerate(order):
        alone = _raw(core, _state(m, core, [models[i]], WS), x, tg)[0]
        assert _same(cut[j], alone), (j, models[i].hidden)
        assert _same(pairs[129 * j:129 * j + 129], alone), j


# ---- 4. statistics --------------------------------------------------------------------------------------------------------------

@gpu
def test_statistics_equal_numpy(fx):
    m = fx.m
    core = fx.core('default')
    F = core.feature_size
    models = [_model(m, F, H, ACTS[i % 4], 500 + i, 'keras 1.3') for i, H in enumerate((20, 64, 128, 9))]
    st = _state(m, core, models, WS)
    x, tg = fx.x, fx.tg
    thr = np.concatenate([[0.5], m.offline.graph_thresholds(m.ListenerParams())]).astype(np.float64)
    thr = np.unique(thr.astype(np.float32)).astype(np.float64)
    res = td._host(core.score_rows(x, tg, st.rows, st.weights, thresholds=thr, miss_threshold=0.5, miss_capacity=5))
    raw = res['raw']
    td._check_stats(res, raw, tg, thr)
    want = np.nonzero((raw > np.float32(0.5)) != (tg[None] != 0))
    assert np.array_equal(res['misses'], np.sort(want[0] * 300 + want[1]))
    # without raw, in workspace batches, and as two calls added up
    core.rows_groups(3, 300)
    try:
        lean = td._host(core.score_rows(x, tg, st.rows, st.weights, thresholds=thr, per_entry=False, miss_threshold=0.5))
    finally:
        core.rows_groups(0, 0)
    for key in ('count', 'hist', 'fit', 'misses'):
        assert np.array_equal(lean[key], res[key]), key
    # (cut at a multiple of 16 clips: entry r keeps pb_predict's place, whose row in a 16-row block decides the last bit)
    a = td._host(core.score_rows(x[:112].contiguous(), tg[:112], st.rows, st.weights, thresholds=thr, per_entry=False))
    b = td._host(core.score_rows(x[112:].contiguous(), tg[112:], st.rows, st.weights, thresholds=thr, per_entry=False))
    for key in ('count', 'hist', 'fit'):
        assert np.array_equal(a[key] + b[key], res[key]), key
    # pairs: random clips, networks interleaved, cut into batches anywhere: raw equals the cross product's entries
    rs = np.random.RandomState(5)
    rows = rs.randint(0, 4, 700).astype(np.int32)
    recs = rs.randint(0, 300, 700).astype(np.int32)
    for nets, cap in ((0, 0), (2, 37), (1, 130)):
        core.rows_groups(nets, cap)
        try:
            p = td._host(core.score_rows(x, tg, st.rows, st.weights, rows, recs, thresholds=thr, miss_threshold=0.5))
            pl = td._host(core.score_rows(x, tg, st.rows, st.weights, rows, recs, thresholds=thr, per_entry=False,
                                          miss_threshold=0.5))
        finally:
            core.rows_groups(0, 0)
        assert _same(p['raw'], raw[rows, recs])
        td._check_stats(p, p['raw'], tg[recs], thr, rows=rows, k=4)
        want = np.nonzero((p['raw'] > np.float32(0.5)) != (tg[recs] != 0))[0]
        assert np.array_equal(p['misses'], want) and np.array_equal(pl['misses'], want)
        for key in ('count', 'hist', 'fit'):
            assert np.array_equal(pl[key], p[key]), key
    # offline.test_rows: DatasetStats and misclassified clips as test_pool reports them
    stats, missed = m.offline.test_rows(core, st, x, tg, thresholds=thr, misses=True)
    for i in range(4):
        assert np.array_equal(stats[i].count, res['count'][i]) and np.array_equal(stats[i].hist, res['hist'][i])
        assert np.array_equal(missed[i], np.nonzero((raw[i] > np.float32(0.5)) != (tg != 0))[0])


# ---- 5. from training -----------------------------------------------------------------------------------------------------------

@gpu
def test_scores_a_trained_state(fx):
    m = fx.m
    clips, tg = train_task.dataset(0, train_task.N_TRAIN)
    t_clips, t_tg = train_task.dataset(10000, train_task.N_TEST)
    core = m.PreciseB200()
    state = m.offline.TrainState.from_models(core, [m.GruModel.init(13, 64, 0), m.GruModel.init(13, 20, 1)], [0, 1])
    assert state.wide
    m.offline.train(core, state, m.offline.vectorize_clips(core, clips), tg, epochs=train_task.EPOCHS, batch_size=train_task.BATCH)
    tx = m.offline.vectorize_clips(core, t_clips)
    stats, missed = m.offline.test_rows(core, state, tx, t_tg, thresholds=(0.25, 0.5), misses=True)
    for i, g in enumerate(state.models()):
        raw = _predict(m, m.ListenerParams(), g, tx)
        if g.hidden == 64:                   # pb_predict runs gru_wide_kernel: the same raw, so the same statistics
            count, hist, fit = td.od.dataset_stats(raw, t_tg, np.float32([0.25, 0.5]))
            assert np.array_equal(stats[i].count, count) and np.array_equal(stats[i].hist, hist)
            assert np.array_equal(missed[i], np.nonzero((raw > 0.5) != (t_tg != 0))[0])
            print('held-out accuracy at H = 64 from the rows: %.3f' % stats[i].accuracy())
            assert stats[i].accuracy() >= train_task.MIN_ACCURACY
    # a fused state (stride 2980) scores too, and agrees with its wide copy
    fused = m.offline.TrainState.from_models(core, [state.models()[1]], [0])
    assert fused.stride == TS
    a = core.score_rows(tx, t_tg, fused.rows, fused.weights)
    b = core.score_rows(tx, t_tg, state.rows, state.weights)
    assert _same(a['raw'].cpu().numpy()[0], b['raw'].cpu().numpy()[1])
    core.close()


# ---- 6. refusals and isolation --------------------------------------------------------------------------------------------------

@gpu
def test_refusals_write_nothing_and_state_is_untouched(fx):
    m, torch = fx.m, fx.torch
    g = m.GruModel.random(13, 20, seed=8, scale=0.1)
    sb = m.StreamBatch(g, 3)
    sb.set_pool(1)
    sb.pool_load(0, g)
    sb.set_stream_pool(np.zeros(3, np.int32))
    rs = np.random.RandomState(1)
    pcm = torch.from_numpy(np.clip(rs.randn(3, 1024) * 3000, -32768, 32767).astype(np.int16)).cuda()
    sb.update_pool(pcm)
    core = sb.core
    before, ids = core.export_streams(n=3).cpu().numpy(), core.stream_pool()
    lib, h = core.lib, core._h
    x, tg = fx.x, np.ascontiguousarray(fx.tg)
    models = [_model(m, 13, 64, ACTS[0], 1), _model(m, 13, 8, ACTS[1], 2)]
    st = _state(m, core, models, WS)
    arr, k = st.rows
    outs = [torch.full(s, 7, dtype=d, device='cuda') for s, d in (((2, 300), torch.float32), ((2, 2), torch.int64),
                                                                  ((2, 2, 3), torch.int64), ((2, 2, 3), torch.int64),
                                                                  ((4,), torch.int64), ((1,), torch.int64))]
    snap = [o.cpu().numpy().copy() for o in outs]
    vp = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    ip = lambda a: np.ascontiguousarray(a, np.int32).ctypes.data_as(C.c_void_p)
    thr1 = np.asarray([0.5], np.float64)

    def call(**kw):
        a = dict(h=h, x=vp(x), n=300, tg=tg.ctypes.data_as(C.c_void_p), rows=arr, k=k, w=vp(st.weights), stride=WS, pr=None,
                 pc=None, np_=0, thr=thr1.ctypes.data_as(C.c_void_p), n_thr=1, raw=vp(outs[0]), count=vp(outs[1]),
                 hist=vp(outs[2]), fit=vp(outs[3]), mt=0.5, miss=vp(outs[4]), cap=4, n_miss=vp(outs[5]))
        a.update(kw)
        return lib.pb_score_rows(a['h'], a['x'], a['n'], a['tg'], a['rows'], a['k'], a['w'], a['stride'], a['pr'], a['pc'],
                                 a['np_'], a['thr'], a['n_thr'], a['raw'], a['count'], a['hist'], a['fit'], a['mt'], a['miss'],
                                 a['cap'], a['n_miss'], None)

    row = lambda H, a=0, r=0: (m.core.pb_train_row * 1)(m.core.pb_train_row(H, a, r, 0))
    down = np.asarray([0.5, 0.4], np.float64)
    invalid = [dict(h=None), dict(stride=TS), dict(stride=0), dict(stride=WS + 1), dict(k=-1), dict(rows=None),
               dict(rows=row(0), k=1), dict(rows=row(129), k=1), dict(rows=row(25), k=1, stride=TS), dict(rows=row(20, 2), k=1),
               dict(rows=row(20, 0, 5), k=1), dict(n=-1), dict(tg=None), dict(w=None), dict(x=None),
               dict(raw=None, count=None, hist=None, fit=None, miss=None, cap=0, n_miss=None),
               dict(pr=ip([0, 1]), pc=None, np_=2), dict(pr=ip([0, 2]), pc=ip([0, 1]), np_=2), dict(pr=ip([0, 1]), pc=ip([0, 300]), np_=2),
               dict(np_=-1), dict(n_thr=-1), dict(n_thr=1025), dict(n_thr=0), dict(thr=None),
               dict(thr=down.ctypes.data_as(C.c_void_p), n_thr=2), dict(cap=-1), dict(miss=None), dict(n_miss=None)]
    for kw in invalid:
        assert call(**kw) == -1, kw
    for params in (m.ListenerParams(use_delta=True), m.ListenerParams(n_filt=20, n_mfcc=17)):
        other = m.PreciseB200(params)
        assert call(h=other._h) == -2
        other.close()
    torch.cuda.synchronize()
    for o, s in zip(outs, snap):
        assert _same(o.cpu().numpy(), s)
    assert call() == 0
    torch.cuda.synchronize()
    assert _same(core.export_streams(n=3).cpu().numpy(), before) and np.array_equal(core.stream_pool(), ids)
    ref = m.StreamBatch(g, 3)
    ref.set_pool(1)
    ref.pool_load(0, g)
    ref.set_stream_pool(np.zeros(3, np.int32))
    ref.update_pool(pcm)
    assert _same(ref.update_pool(pcm)['raw'].cpu().numpy(), sb.update_pool(pcm)['raw'].cpu().numpy())


# ---- 7. the command -------------------------------------------------------------------------------------------------------------

@gpu
def test_command_with_wide_networks(fx, tmp_path, capsys):
    m = fx.m
    from mycroft_precise_b200 import test as ptest
    from mycroft_precise_b200.model_io import save_weights
    from mycroft_precise_b200.params import ListenerParams, save_params
    data = tmp_path / 'data'
    for i in range(24):
        tw._write(str(data / 'test' / ('wake-word' if i % 2 == 0 else 'not-wake-word') / ('t%02d.wav' % i)),
                  train_task.clip(700 + i, i % 2 == 0))
    names, models = [], []
    # the 20-unit network has tanh / sigmoid, so that pb_predict scores it on gru_wide_kernel too (the default pair would
    # take its own kernels) and every expected block comes from pb_predict
    for H, seed, act in ((20, 1, ACTS[1]), (64, 2, ACTS[0]), (128, 3, ACTS[0])):
        g = _model(m, 13, H, act, seed, 'keras 1.3')
        n = str(tmp_path / ('n%d.npz' % H))
        save_weights(n, g)
        save_params(n, ListenerParams())
        names.append(n)
        models.append(g)
    core = m.PreciseB200()
    files, clips, targets = ptest.load_folder(str(data), False)
    x = m.offline.vectorize_clips(core, clips)
    for flags in ([], ['-nf'], ['--calc-threshold']):
        ptest.main(names + [str(data)] + flags)
        got = capsys.readouterr().out
        want = []
        for name, g in zip(names, models):
            raw = _predict(m, ListenerParams(), g, x)
            count, hist, fit = td.od.dataset_stats(raw, targets, np.float32([0.5]))
            stv = m.offline.DatasetStats([0.5], count, hist, fit)
            miss = np.nonzero((raw > np.float32(0.5)) != (targets != 0))[0]
            want.append('=== %s ===' % name)
            if '-nf' not in flags:
                want += ['=== False Positives ===', '\n'.join(files[i] for i in miss if not targets[i]), '',
                         '=== False Negatives ===', '\n'.join(files[i] for i in miss if targets[i]), '']
            want += [stv.counts_str(0.5), '', stv.summary_str(0.5)]
            if '--calc-threshold' in flags:
                fit2 = m.offline.calc_threshold(stv)
                want.append('No data (or all NaN)' if fit2 is None else 'Peak: {:.2f} mu, {:.2f} std'.format(*fit2))
        assert got == '\n'.join(want) + '\n', flags
    # a wide set with deltas, or a feature size above 16, is refused before any device work
    for params, F in ((ListenerParams(use_delta=True), 26), (ListenerParams(n_filt=20, n_mfcc=17), 17)):
        bad = str(tmp_path / ('bad%d.npz' % F))
        save_weights(bad, m.GruModel.random(F, 20, seed=1))
        save_params(bad, params)
        with pytest.raises(ValueError, match='hidden <= 128, feature size <= 16 and no deltas|front end differs'):
            ptest.main([names[1], bad, str(data)])
    core.close()
