"""Training of networks up to 128 GRU units on the device (pb_train_wide, pb_train_wide_loss; PreciseB200.train / train_loss on
rows of PB_TRAIN_WIDE_STRIDE, offline.TrainState's wide layout, offline.train and train_generated on it, and the train and
train_generated commands) against the float64 restatement of oracle/train.py at the wide stride (tests/train_wide_oracle.py).

- Gradients block by block with test_gpu_train_sweep's yardstick (check_grad): max |g_dev - g64| <= 10 max |g32 - g64| +
  1e-6 max |g64|, 1e-5 for one-element blocks and hard_sigmoid's jump where a pre-activation lies within 1e-4 of +-2.5.
  Hidden sizes 1 .. 128 around the fragment tiles of 8 and 16, all four activation pairs, dropout 0 and 0.5, the sweep's
  three weight families, 1 to 129 entries per row, on six front ends.
- Against pb_train at H <= 24 within the same yardstick; RMSprop's step; three epochs and batch size 1 against train_row.
- Bit-for-bit determinism across runs, row order, epoch splitting, workspace groups and state launches.
- Refusals, untouched buffers, streams and pool; the largest accepted row; the chirp task at H = 64 scored by the wide scan;
  augment= and train_generated against their hand-written loops; the commands.

-m gpu throughout.  The per-front-end worst errors are printed (pytest -s) as "wide sweep:" lines."""
import ctypes as C
import os
import sys
import wave

import numpy as np
import pytest

from oracle import train as ot

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_train_sweep as sw  # noqa: E402
import train_task  # noqa: E402
import train_wide_oracle as wo  # noqa: E402

gpu = pytest.mark.gpu
WS = wo.WIDE_STRIDE
HIDDEN = (1, 8, 16, 17, 24, 25, 31, 32, 33, 48, 64, 100, 120, 127, 128)
HIDDEN_SOME = (1, 17, 25, 64, 127, 128)
COUNTS = (1, 5, 16, 17, 63, 64, 65, 129)
FRONTS = ('default', 'f16', 'f1', 'mels16', 't1', 't112')


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


@pytest.fixture(scope='module')
def fx():
    pytest.importorskip('torch')
    f = sw.Fixture()
    yield f
    f.close()


def _oracle(specs, w, x, y, recs_of, F, rate, epoch, bias, masks, dtype, kink=0.0):
    out = []
    for i, (H, a, r, s) in enumerate(specs):
        recs = recs_of[i]
        m = masks(s, epoch, len(recs), F, rate)
        out.append(wo.loss_grad(w[i].astype(dtype), F, H, x[recs].astype(dtype), y[recs].astype(dtype), m.astype(dtype), bias,
                                a, r, dtype, kink)[:2] if kink == 0 or r == 'hard_sigmoid' else None)
    return out


def _jumps(specs, w, x, y, recs_of, F, rate, epoch, bias, masks):
    wide = _oracle(specs, w, x, y, recs_of, F, rate, epoch, bias, masks, np.float64, sw.KINK)
    narrow = _oracle(specs, w, x, y, recs_of, F, rate, epoch, bias, masks, np.float64, -sw.KINK)
    return [None if p is None else (p[1], q[1]) for p, q in zip(wide, narrow)]


def _rows(core, specs):
    return core.train_rows(*[[s[c] for s in specs] for c in range(4)])


def _random_rows(specs, F, seed, scale=0.3):
    w = np.zeros((len(specs), WS), np.float32)
    for i, sp in enumerate(specs):
        n = ot.row_size(F, sp[0])
        w[i, :n] = np.random.RandomState(seed + i).randn(n) * scale
    return w


# ---- 1. gradients against float64 --------------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize('front', FRONTS)
def test_gradient_sweep(fx, front):
    core = fx.core(front)
    F, T = core.feature_size, core.n_features
    hidden = HIDDEN if front == 'default' else HIDDEN_SOME
    x = np.random.RandomState(1).randn(160, T, F).astype(np.float32) * 2
    y = (np.random.RandomState(2).rand(len(x)) < 0.4).astype(np.uint8)
    dx = fx.dev(x)
    specs0 = [(H, a, r) for (a, r) in sw.ACTS for H in hidden]
    counts = [COUNTS[i % len(COUNTS)] for i in range(len(specs0))]
    pr_, pc_, recs_of = sw.rows_of(counts, len(x), 3)
    masks = sw.Masks()
    bad = []
    for family in sw.FAMILIES:
        models = [sw._model(family, F, H, (a, r), 50 + i) for i, (H, a, r) in enumerate(specs0)]
        specs = [(H, act[0], act[1], 900 + i) for i, ((H, _a, _r), (_g, act)) in enumerate(zip(specs0, models))]
        w = sw.padded(np.stack([wo.pack(mo) for mo, _ in models]), specs, F)
        dw = fx.dev(w)
        rows = _rows(core, specs)
        for rate in (0.0, 0.5):
            loss, grad = core.train_loss(dx, y, rows, dw, pr_, pc_, loss_bias=0.8, dropout=rate, epoch=3, grad=True)
            loss, grad = loss.cpu().numpy(), grad.cpu().numpy()
            want = _oracle(specs, w, x, y, recs_of, F, rate, 3, 0.8, masks, np.float64)
            f32 = _oracle(specs, w, x, y, recs_of, F, rate, 3, 0.8, masks, np.float32)
            jump = _jumps(specs, w, x, y, recs_of, F, rate, 3, 0.8, masks)
            worst = 0.0
            for i, (H, a, r, s) in enumerate(specs):
                what = (front, family, rate, H, a, r, counts[i])
                sw.check_loss(loss[i], want[i][0], f32[i][0], what)
                for name, (err, spread, top) in sw.check_grad(grad[i], want[i][1], f32[i][1], F, H, what, jump[i], bad).items():
                    worst = max(worst, err / spread if spread > 0 else 0.0)
            assert sw.pad_ok(dw.cpu().numpy(), specs, F)
            print('wide sweep: %s | %s | dropout %.1f | worst ratio |g_dev - g64| / |g32 - g64| %.3g' % (front, family, rate, worst))
    assert not bad, bad[:20]


@gpu
def test_agrees_with_pb_train_up_to_24_units(fx):
    core = fx.core('default')
    F, T = core.feature_size, core.n_features
    specs = [(H, a, r, 7 + i) for i, (a, r) in enumerate(sw.ACTS) for H in (1, 8, 17, 24)]
    x = np.random.RandomState(4).randn(100, T, F).astype(np.float32)
    y = (np.random.RandomState(5).rand(100) < 0.5).astype(np.uint8)
    counts = [COUNTS[i % len(COUNTS)] for i in range(len(specs))]
    pr_, pc_, recs_of = sw.rows_of(counts, len(x), 6)
    w = _random_rows(specs, F, 30)
    rows = _rows(core, specs)
    masks = sw.Masks()
    for rate in (0.0, 0.5):
        _, gw = core.train_loss(fx.dev(x), y, rows, fx.dev(w), pr_, pc_, dropout=rate, epoch=1, grad=True)
        _, gf = core.train_loss(fx.dev(x), y, rows, fx.dev(np.ascontiguousarray(w[:, :ot.STRIDE])), pr_, pc_, dropout=rate,
                                epoch=1, grad=True)
        gw, gf = gw.cpu().numpy(), gf.cpu().numpy()
        want = _oracle(specs, w, x, y, recs_of, F, rate, 1, 0.8, masks, np.float64)
        f32 = _oracle(specs, w, x, y, recs_of, F, rate, 1, 0.8, masks, np.float32)
        jump = _jumps(specs, w, x, y, recs_of, F, rate, 1, 0.8, masks)
        for i, sp in enumerate(specs):
            g_f = np.zeros(WS, np.float32)
            g_f[:ot.STRIDE] = gf[i]
            # the fused gradient takes the float64 one's place: the two kernels agree within the yardstick
            sw.check_grad(gw[i], g_f.astype(np.float64), f32[i][1] - want[i][1] + g_f, F, sp[0], ('vs pb_train', rate) + sp,
                          jump[i])


# ---- 2. optimizer and epochs ---------------------------------------------------------------------------------------------------

@gpu
def test_rmsprop_step_and_epochs_follow_float64(fx):
    torch = fx.torch
    core = fx.core('default')
    F, T = core.feature_size, core.n_features
    x = np.random.RandomState(8).randn(48, T, F).astype(np.float32)
    y = (np.arange(48) % 3 == 0).astype(np.uint8)
    spec = [(40, 'tanh', 'hard_sigmoid', 11)]
    w = _random_rows(spec, F, 12, 0.2)
    rows = _rows(core, spec)
    # one entry, one step at non-default lr, rho, epsilon: the update is the formula on the call's own gradient
    pr_, pc_ = np.zeros(1, np.int32), np.asarray([5], np.int32)
    _, g = core.train_loss(fx.dev(x), y, rows, fx.dev(w), pr_, pc_, loss_bias=0.7, dropout=0.3, epoch=4, grad=True)
    g = g.cpu().numpy()[0]
    dw, drms = fx.dev(w), torch.zeros((1, WS), dtype=torch.float32, device='cuda')
    core.train(fx.dev(x), y, rows, dw, drms, pr_, pc_, epochs=1, epoch0=4, batch_size=3, lr=0.01, rho=0.8, epsilon=1e-4,
               loss_bias=0.7, dropout=0.3)
    a = np.float32(1 - np.float32(0.8)) * (g * g)
    want = w[0] - np.float32(0.01) * g / (np.sqrt(a) + np.float32(1e-4))
    assert _same(drms.cpu().numpy()[0], a)
    assert np.allclose(dw.cpu().numpy()[0], want, rtol=1e-6, atol=1e-9)
    # three epochs at batch sizes 16 and 1 (batch 1 checks the shuffle order and masks) against train_row in float64
    n = ot.row_size(F, 40)
    for bs, epochs in ((16, 3), (1, 1)):
        dw, drms = fx.dev(w), torch.zeros((1, WS), dtype=torch.float32, device='cuda')
        loss = core.train(fx.dev(x), y, rows, dw, drms, epochs=epochs, batch_size=bs).cpu().numpy()[0]
        row, rms = w[0].astype(np.float64), np.zeros(WS)
        want = wo.train_row(row, rms, F, 40, x.astype(np.float64), y.astype(np.float64), np.arange(48), 11, epochs,
                            batch_size=bs, activation='tanh')
        got = dw.cpu().numpy()[0]
        # RMSprop moves each weight by about lr per step whatever the gradient's size, so float32 rounding of a tiny
        # gradient can flip a step: the bound is on the 99th percentile, as test_gpu_generated's
        d = np.abs(got[:n] - row[:n])
        assert np.allclose(loss, want, rtol=1e-4), (bs, loss, want)
        assert np.quantile(d, 0.99) < 1e-4 and d.max() < 3 * 0.001 * epochs * (48 // bs), (bs, np.quantile(d, 0.99), d.max())
        assert not np.any(got[n:])


# ---- 3. determinism --------------------------------------------------------------------------------------------------------------

@gpu
def test_bit_for_bit_determinism(fx):
    torch = fx.torch
    core = fx.core('default')
    F, T = core.feature_size, core.n_features
    n_rec = 1000
    x = np.random.RandomState(9).randn(n_rec, T, F).astype(np.float32)
    y = (np.random.RandomState(10).rand(n_rec) < 0.3).astype(np.uint8)
    dx = fx.dev(x)
    # 80 rows of 1 000 entries at batch 1 000: 16 partial rows each, about 3.6 MB per row at H = 25 -> two workspace
    # groups, and 1 280 tiles of 1.5 MB of state per batch -> four state launches
    specs = [((25, 32, 64, 128)[i % 4] if i < 4 else 25, sw.ACTS[i % 4][0], sw.ACTS[i % 4][1], 300 + i) for i in range(80)]
    w = _random_rows(specs, F, 40, 0.2)

    def fit(idx, epochs=2, calls=1):
        sp = [specs[i] for i in idx]
        dw, drms = fx.dev(w[idx]), torch.zeros((len(idx), WS), dtype=torch.float32, device='cuda')
        losses = [core.train(dx, y, _rows(core, sp), dw, drms, epochs=epochs // calls, epoch0=c * (epochs // calls),
                             batch_size=1000) for c in range(calls)]
        return dw.cpu().numpy(), drms.cpu().numpy(), torch.cat(losses, 1).cpu().numpy()

    order = np.random.RandomState(11).permutation(80)
    a = fit(order)
    b = fit(order)
    assert all(_same(p, q) for p, q in zip(a, b))
    c = fit(order, calls=2)
    assert all(_same(p, q) for p, q in zip(a, c))
    for j in (0, 1, 2, 3, 50):                     # one launch, one group
        alone = fit([j])
        i = int(np.where(order == j)[0][0])
        assert all(_same(p[i], q[0]) for p, q in zip(a, alone)), j


# ---- 4. refusals and what accepted calls leave alone ----------------------------------------------------------------------------

@gpu
def test_refused_calls_change_nothing(fx):
    m = fx.m
    torch = fx.torch
    core = fx.core('default')
    lib, h = core.lib, core._h
    F, T = core.feature_size, core.n_features
    x = np.random.RandomState(3).randn(400, T, F).astype(np.float32)
    dx = fx.dev(x)
    specs = [(64, 'linear', 'hard_sigmoid', 1), (8, 'tanh', 'sigmoid', 2)]
    arr, k = _rows(core, specs)
    w = _random_rows(specs, F, 1)
    dw = fx.dev(w)
    drms = torch.full_like(dw, 0.5)
    dloss = torch.zeros((k, 2), dtype=torch.float64, device='cuda')
    w0, r0 = dw.cpu().numpy().copy(), drms.cpu().numpy().copy()
    tg = np.ascontiguousarray((np.arange(400) % 2).astype(np.uint8))
    vp = lambda t: C.c_void_p(t.data_ptr())
    tp = tg.ctypes.data_as(C.c_void_p)
    pc = np.asarray([0, 1, 2], np.int32)
    pc_bad = np.asarray([0, 1, 400], np.int32)
    o = m.core.pb_train_opts()
    assert lib.pb_train_opts_default(C.byref(o)) == 0

    def train(opts=o, **kw):
        a = dict(h=h, x=vp(dx), n=400, tg=tp, rows=arr, k=k, pr=None, pc=None, np_=0, w=vp(dw), rms=vp(drms), loss=vp(dloss))
        a.update(kw)
        return lib.pb_train_wide(a['h'], a['x'], a['n'], a['tg'], a['rows'], a['k'], a['pr'], a['pc'], a['np_'],
                                 C.byref(opts) if opts is not None else None, a['w'], a['rms'], a['loss'], None)

    def opts(**kw):
        x = m.core.pb_train_opts()
        lib.pb_train_opts_default(C.byref(x))
        for key, v in kw.items():
            setattr(x, key, v)
        return x

    row = lambda H, a=0: (m.core.pb_train_row * 1)(m.core.pb_train_row(H, a, 0, 0))
    ip = lambda a: np.asarray(a, np.int32).ctypes.data_as(C.c_void_p)
    refusals = [dict(h=None), dict(opts=None), dict(x=None), dict(tg=None), dict(rows=None), dict(k=-1), dict(n=-1),
                dict(w=None), dict(rms=None), dict(rows=row(0), k=1), dict(rows=row(129), k=1), dict(rows=row(20, 2), k=1),
                dict(pr=ip([0, 1, 2]), pc=None, np_=3), dict(pr=ip([0, 1, 2]), pc=pc.ctypes.data_as(C.c_void_p), np_=3),
                dict(pr=ip([0, 1, 1]), pc=pc_bad.ctypes.data_as(C.c_void_p), np_=3), dict(np_=-1, pr=ip([0]), pc=ip([0])),
                dict(opts=opts(epochs=0)), dict(opts=opts(epoch0=-1)), dict(opts=opts(batch_size=0)),
                dict(opts=opts(lr=float('nan'))), dict(opts=opts(lr=-1.0)), dict(opts=opts(rho=1.0)), dict(opts=opts(rho=-0.1)),
                dict(opts=opts(epsilon=-1.0)), dict(opts=opts(epsilon=float('inf'))), dict(opts=opts(loss_bias=1.5)),
                dict(opts=opts(dropout=1.0)), dict(opts=opts(dropout=-0.1))]
    for kw in refusals:
        assert train(**kw) == -1, kw
    L = lambda **kw: lib.pb_train_wide_loss(h, vp(dx), 400, tp, kw.get('rows', arr), kw.get('k', k), None, None, 0,
                                            kw.get('bias', 0.8), kw.get('rate', 0.0), kw.get('epoch', 0), kw.get('w', vp(dw)),
                                            kw.get('loss', vp(dloss)), None, None)
    assert L(epoch=-1) == -1 and L(loss=None) == -1 and L(bias=-0.1) == -1 and L(rate=1.0) == -1 and L(w=None) == -1
    assert L(rows=row(129), k=1) == -1 and L(rows=row(0), k=1) == -1
    # front ends outside pb_vectorize_clips' range: deltas, and 113 steps
    for params in (m.ListenerParams(use_delta=True), m.ListenerParams(buffer_t=5.7)):
        other = m.PreciseB200(params)
        assert params.use_delta or other.n_features == 113
        ox = torch.zeros((4, other.n_features, other.feature_size), dtype=torch.float32, device='cuda')
        orows = other.train_rows([64], ['linear'], ['hard_sigmoid'], [0])
        assert lib.pb_train_wide(other._h, vp(ox), 4, tp, orows[0], 1, None, None, 0, C.byref(o), vp(dw), vp(drms), None,
                                 None) == -2
        assert lib.pb_train_wide_loss(other._h, vp(ox), 4, tp, orows[0], 1, None, None, 0, 0.8, 0.0, 0, vp(dw), vp(dloss),
                                      None, None) == -2
        other.close()
    torch.cuda.synchronize()
    assert _same(dw.cpu().numpy(), w0) and _same(drms.cpu().numpy(), r0)


@gpu
def test_training_leaves_streams_and_pool_alone(fx):
    m = fx.m
    torch = fx.torch
    g = m.GruModel.random(13, 20, seed=8, scale=0.1)
    sb = m.StreamBatch(g, 3)
    sb.set_pool(1)
    sb.pool_load(0, g)
    sb.set_stream_pool(np.zeros(3, np.int32))
    rs = np.random.RandomState(1)
    pcm = torch.from_numpy(np.clip(rs.randn(3, 1024) * 3000, -32768, 32767).astype(np.int16)).cuda()
    sb.update_pool(pcm)
    core = sb.core
    before = core.export_streams(n=3).cpu().numpy()
    ids = core.stream_pool()
    x = torch.from_numpy(rs.randn(20, core.n_features, core.feature_size).astype(np.float32)).cuda()
    specs = [(96, 'linear', 'hard_sigmoid', 1)]
    w = _random_rows(specs, core.feature_size, 2)
    core.train(x, np.arange(20) % 2, _rows(core, specs), fx.dev(w), torch.zeros((1, WS), dtype=torch.float32, device='cuda'),
               epochs=2, batch_size=8)
    core.train_loss(x, np.arange(20) % 2, _rows(core, specs), fx.dev(w), grad=True)
    torch.cuda.synchronize()
    assert _same(core.export_streams(n=3).cpu().numpy(), before)
    assert np.array_equal(core.stream_pool(), ids)
    ref = m.StreamBatch(g, 3)
    ref.set_pool(1)
    ref.pool_load(0, g)
    ref.set_stream_pool(np.zeros(3, np.int32))
    ref.update_pool(pcm)
    assert _same(ref.update_pool(pcm)['raw'].cpu().numpy(), sb.update_pool(pcm)['raw'].cpu().numpy())
    # the pool holds the fused family: pool_train refuses a wide network before training anything
    with pytest.raises(ValueError, match='at most 24 units'):
        sb.pool_train([0], [m.GruModel.init(13, 32, 0)], [train_task.clip(0, True)], [1])


@gpu
def test_largest_accepted_row(fx):
    torch = fx.torch
    core = fx.core('t112')
    assert core.n_features == 112
    m = fx.m
    core16 = m.PreciseB200(m.ListenerParams(buffer_t=5.65, n_mfcc=16))
    assert (core16.n_features, core16.feature_size) == (112, 16)
    F, T = 16, 112
    x = torch.randn((5000, T, F), device='cuda', generator=torch.Generator('cuda').manual_seed(0))
    y = (np.arange(5000) % 4 == 0).astype(np.uint8)
    specs = [(128, 'tanh', 'sigmoid', 5)]
    w = _random_rows(specs, F, 3, 0.05)
    dw, drms = fx.dev(w), torch.zeros((1, WS), dtype=torch.float32, device='cuda')
    loss = core16.train(x, y, _rows(core16, specs), dw, drms, epochs=1, batch_size=5000).cpu().numpy()
    got = dw.cpu().numpy()[0]
    assert np.all(np.isfinite(loss)) and np.all(np.isfinite(got))
    assert np.any(got[:ot.row_size(F, 128)] != w[0, :ot.row_size(F, 128)]) and not np.any(got[ot.row_size(F, 128):])
    core16.close()


# ---- 5. end to end ---------------------------------------------------------------------------------------------------------------

@gpu
def test_chirp_task_at_64_units_scored_by_the_wide_scan(fx):
    m = fx.m
    clips, tg = train_task.dataset(0, train_task.N_TRAIN)
    t_clips, t_tg = train_task.dataset(10000, train_task.N_TEST)
    core = m.PreciseB200()
    init = m.GruModel.init(13, 64, 0)
    state = m.offline.TrainState.from_models(core, [init], [0])
    assert state.wide and state.weights.shape == (1, WS)
    loss, val = m.offline.train(core, state, m.offline.vectorize_clips(core, clips), tg, epochs=train_task.EPOCHS,
                                batch_size=train_task.BATCH, validation=(m.offline.vectorize_clips(core, t_clips), t_tg))
    assert loss.shape == val.shape == (1, train_task.EPOCHS) and val[0, -1] < val[0, 0]
    trained = state.models()[0]
    assert trained.hidden == 64
    scorer = m.PreciseB200(hidden=64)
    scorer.load_weights(trained.kernel, trained.recurrent, trained.bias, trained.dense_w, trained.dense_b)
    raw = scorer.predict(m.offline.vectorize_clips(core, t_clips)).cpu().numpy().reshape(-1)
    acc = float(np.mean((raw > 0.5) == (t_tg != 0)))
    print('held-out accuracy at H = 64: %.3f' % acc)
    assert acc >= train_task.MIN_ACCURACY
    scorer.close()
    core.close()


@gpu
def test_augment_and_generated_are_their_hand_written_loops(fx):
    m, torch = fx.m, fx.torch
    core = fx.core('default')
    F, T = core.feature_size, core.n_features
    clips, tg = train_task.dataset(0, 24)
    rs = np.random.RandomState(31)
    noise = [np.clip(np.round(rs.randn(50000) * 1000), -32768, 32767).astype(np.int16)]
    init = [m.GruModel.init(F, 40, 0), m.GruModel.init(F, 8, 1)]
    st = m.offline.TrainState.from_models(core, init, [3, 4])
    assert st.wide
    aug = m.offline.Augment(m.offline.NoiseSource(core, noise, 123), 2, 0.05, 0.5, seed=9)
    la = m.offline.train(core, st, clips, tg, epochs=2, batch_size=7, augment=aug)
    ref = m.offline.TrainState.from_models(core, init, [3, 4])
    clean = m.offline.vectorize_clips(core, clips)
    total = sum(len(c) for c in clips)
    src = m.offline.NoiseSource(core, noise, 123)
    items = np.repeat(np.arange(len(clips)), 2)
    losses = []
    for e in range(2):
        u = np.asarray([(ot.key(9, e, i, 0) >> 11) * 2.0 ** -53 for i in range(items.size)])
        src.pos = (123 + e * 2 * total) % len(src)
        noisy = m.offline.vectorize_noisy(core, clips, src, 0.05 + 0.45 * u, items).view(len(clips), 2, T, F)
        x = torch.cat([clean[:, None], noisy], 1).reshape(-1, T, F).contiguous()
        losses.append(core.train(x, np.repeat(tg, 3), ref.rows, ref.weights, ref.rms, epochs=1, epoch0=e, batch_size=7))
    assert _same(st.weights.cpu().numpy(), ref.weights.cpu().numpy())
    assert _same(torch.cat(losses, 1).cpu().numpy(), la)
    # train_generated: one pb_train_wide epoch per generated epoch
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import test_gpu_generated as tg_mod
    st = m.offline.TrainState.from_models(core, init, [3, 4])
    lg = m.offline.train_generated(core, st, tg_mod._task_generator(core), 2, steps_per_epoch=3, batch_size=40)
    ref = m.offline.TrainState.from_models(core, init, [3, 4])
    gen = tg_mod._task_generator(core)
    losses = []
    for e in range(2):
        gen.seek(e * 120)
        x, y, _, _ = gen.run(gen.plan(120))
        losses.append(core.train(x, y, ref.rows, ref.weights, ref.rms, epochs=1, epoch0=e, batch_size=40, loss_bias=0.8,
                                 dropout=0.2))
    assert _same(st.weights.cpu().numpy(), ref.weights.cpu().numpy())
    assert _same(torch.cat(losses, 1).cpu().numpy(), lg)


# ---- 6. commands -----------------------------------------------------------------------------------------------------------------

def _write(path, pcm):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with wave.open(path, 'wb') as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(16000)
        w.writeframes(np.ascontiguousarray(pcm, '<i2').tobytes())


@gpu
def test_commands_train_wide_networks(fx, tmp_path, capsys, monkeypatch):
    from mycroft_precise_b200 import train as ptrain
    from mycroft_precise_b200 import train_generated as pgen
    from mycroft_precise_b200.model_io import GruModel, load_weights, save_weights
    from mycroft_precise_b200.params import ListenerParams, save_params
    data, rnd = tmp_path / 'data', tmp_path / 'random'
    for i in range(30):
        _write(str(data / ('wake-word' if i % 2 == 0 else 'not-wake-word') / ('c%03d.wav' % i)), train_task.clip(i, i % 2 == 0))
    for i in range(6):
        _write(str(data / 'test' / ('wake-word' if i % 2 == 0 else 'not-wake-word') / ('t%d.wav' % i)),
               train_task.clip(500 + i, i % 2 == 0))
    rs = np.random.RandomState(2)
    for i in range(4):
        _write(str(rnd / ('bg%d.wav' % i)), np.clip(rs.randn(150000) * 600, -32768, 32767).astype(np.int16))
    a, b = str(tmp_path / 'a.npz'), str(tmp_path / 'b.npz')
    ptrain.main([a, b, str(data), '-e', '2', '-b', '16', '--hidden', '64'])
    text = capsys.readouterr().out
    assert text.count('Epoch 2/2 - loss: ') == 2 and 'val_loss' in text
    for n in (a, b):
        assert os.path.isfile(n) and os.path.isfile(n + '.params') and load_weights(n).hidden == 64
    # an existing 32-unit network is fine-tuned
    c = str(tmp_path / 'c.npz')
    m32 = GruModel.init(13, 32, 5)
    save_weights(c, m32)
    save_params(c, ListenerParams())
    ptrain.main([c, str(data), '-e', '1', '-b', '16'])
    tuned = load_weights(c)
    assert 'Epoch 1/1 - loss: ' in capsys.readouterr().out
    assert tuned.hidden == 32 and not np.array_equal(tuned.recurrent, m32.recurrent)
    monkeypatch.chdir(tmp_path)
    g = str(tmp_path / 'g.npz')
    pgen.main([g, str(data), '-r', str(rnd), '-e', '1', '-t', '3', '-b', '40', '--hidden', '48'])
    assert 'Epoch 1/1 - loss: ' in capsys.readouterr().out
    assert load_weights(g).hidden == 48 and open(str(tmp_path / 'g.epoch')).read() == '1'
    with pytest.raises(ValueError, match='hidden <= 128'):
        ptrain.main([str(tmp_path / 'd.npz'), str(data), '-e', '1', '--hidden', '129'])
