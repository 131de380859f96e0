"""Training on the device (pb_vectorize_clips, pb_train, pb_train_loss; PreciseB200.vectorize_clips / train / train_loss,
offline.vectorize_clips / TrainState / train, StreamBatch.pool_train, python -m mycroft_precise_b200.train), against the
float64 restatement in oracle/train.py.  -m gpu."""
import ctypes as C
import os
import sys
import wave

import numpy as np
import pytest

from oracle import gru as og
from oracle import mfcc as om
from oracle import train as ot
from oracle.params import OracleParams

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import train_task  # noqa: E402

gpu = pytest.mark.gpu
PAIRS = [('linear', 'hard_sigmoid'), ('tanh', 'sigmoid'), ('linear', 'sigmoid'), ('tanh', 'hard_sigmoid')]
F, T = 13, 29


def _noise(n, seed, sigma=3000):
    rs = np.random.RandomState(seed)
    return np.clip(rs.randn(n) * sigma * (1 + np.sin(np.arange(n) / 4000.0)), -32768, 32767).astype(np.int16)


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


class Fixture:
    def __init__(self):
        import torch
        import mycroft_precise_b200 as m
        self.m, self.torch = m, torch
        self.core = m.PreciseB200()
        rs = np.random.RandomState(3)
        self.x = rs.randn(400, T, F).astype(np.float32)
        self.y = (rs.rand(400) < 0.4).astype(np.uint8)
        self.dx = torch.from_numpy(self.x).cuda()

    def rows(self, specs):
        """specs: (hidden, activation, recurrent_activation, seed) per row -> (ctypes rows, weights [k, STRIDE] float32)."""
        w = np.zeros((len(specs), ot.STRIDE), np.float32)
        for i, (H, a, r, s) in enumerate(specs):
            w[i, :ot.row_size(F, H)] = np.random.RandomState(100 + s).randn(ot.row_size(F, H)) * 0.3
        rows = self.core.train_rows([s[0] for s in specs], [s[1] for s in specs], [s[2] for s in specs], [s[3] for s in specs])
        return rows, w

    def dev(self, a):
        return self.torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.fixture(scope='module')
def fx():
    pytest.importorskip('torch')
    f = Fixture()
    yield f
    f.core.close()


def _pack(clips, lead=0):
    parts = ([_noise(lead, 999)] if lead else []) + list(clips)
    offsets = np.concatenate([[0], np.cumsum([len(c) for c in parts])]).astype(np.int64)
    return np.concatenate(parts), offsets


# ---- 1. inputs ---------------------------------------------------------------------------------------------------------------

@gpu
def test_vectorize_clips_is_the_scored_window(fx):
    """The rows are the window score_dataset scores (pb_predict of them on the tensor-core scan gives the same raw bit for
    bit) and the float64 vectorize of the cropped clip."""
    m = fx.m
    lens = [1, 511, 1599, 1600, 24000, 24001, 30001]
    clips = [_noise(n, 20 + i) for i, n in enumerate(lens)]
    pcm, offsets = _pack(clips, lead=3)
    dpcm = fx.dev(pcm)
    core = m.PreciseB200()
    g = m.GruModel.random(13, 20, seed=4, scale=0.1)
    core.load_weights(g.kernel, g.recurrent, g.bias, g.dense_w, g.dense_b)
    core.set_pool(1)
    core.pool_load(0, g)
    inputs = core.vectorize_clips(dpcm, offsets)
    assert tuple(inputs.shape) == (len(lens) + 1, T, F)
    raw = core.score_dataset(dpcm, offsets, np.ones(len(lens) + 1, np.uint8), np.zeros(1, np.int32))['raw'].cpu().numpy()[0]
    core.gru_mode(2)
    pred = core.predict(inputs).cpu().numpy().reshape(-1)
    assert _same(pred, raw)
    got = inputs.cpu().numpy()[1:]
    opr = OracleParams()
    for j, c in enumerate(clips):
        want = om.vectorize(c.astype(np.float64) / 32767.0, opr)
        assert np.allclose(got[j], want, rtol=1e-4, atol=1e-3), (lens[j], np.max(np.abs(got[j] - want)))
    # offline.vectorize_clips packs the clips its own way (aligned clips may take the fast K1 there): the same rows to the
    # last bits
    alt = m.offline.vectorize_clips(core, clips).cpu().numpy()
    assert alt.shape == got.shape and np.max(np.abs(alt - got)) < 1e-5
    core.close()


# ---- 2. gradients ------------------------------------------------------------------------------------------------------------

def _oracle(fx, specs, w, recs_of, rate, epoch, bias=0.8, dtype=np.float64):
    out = []
    for i, (H, a, r, s) in enumerate(specs):
        recs = recs_of[i]
        m = ot.masks(s, epoch, range(len(recs)), F, rate)
        xx = fx.x[recs].astype(dtype)
        out.append(ot.loss_grad(w[i].astype(dtype), F, H, xx, fx.y[recs].astype(dtype), m.astype(dtype), bias, a, r, dtype)[:2])
    return out


@gpu
@pytest.mark.parametrize('act,ract', PAIRS)
@pytest.mark.parametrize('rate', [0.0, 0.3])
def test_train_loss_gradient_equals_float64(fx, act, ract, rate):
    """Loss and gradient of pb_train_loss against float64, with the bound 10x the float32 restatement's spread from float64
    (plus 1e-6 of the gradient's size), for H in 1, 8, 20, 24 and 1, 70 and 300 entries (pairs)."""
    specs = [(H, act, ract, 7 + H) for H in (1, 8, 20, 24)]
    rows, w = fx.rows(specs)
    counts = [1, 70, 300, 70]
    pr = np.concatenate([np.full(c, i, np.int32) for i, c in enumerate(counts)])
    rs = np.random.RandomState(9)
    pc = rs.randint(0, 400, pr.size).astype(np.int32)
    recs_of = [pc[pr == i] for i in range(len(specs))]
    loss, grad = fx.core.train_loss(fx.dx, fx.y, rows, fx.dev(w), pr, pc, dropout=rate, epoch=2, grad=True)
    loss, grad = loss.cpu().numpy(), grad.cpu().numpy()
    want = _oracle(fx, specs, w, recs_of, rate, 2)
    f32 = _oracle(fx, specs, w, recs_of, rate, 2, dtype=np.float32)
    for i, (H, *_r) in enumerate(specs):
        n = ot.row_size(F, H)
        l64, g64 = want[i]
        l32, g32 = f32[i]
        spread = np.max(np.abs(g32.astype(np.float64) - g64))
        bound = 10 * spread + 1e-6 * np.max(np.abs(g64))
        assert np.max(np.abs(grad[i, :n] - g64[:n])) <= bound, (H, np.max(np.abs(grad[i, :n] - g64[:n])), bound)
        assert not np.any(grad[i, n:])
        assert abs(loss[i] - l64) <= 10 * abs(float(l32) - l64) + 1e-6 * abs(l64), (H, loss[i], l64, l32)


# ---- 3. training ---------------------------------------------------------------------------------------------------------------

@gpu
def test_one_step_and_a_few_epochs_follow_float64(fx):
    specs = [(20, 'linear', 'hard_sigmoid', 1), (12, 'tanh', 'sigmoid', 2)]
    rows, w = fx.rows(specs)
    n = 64
    torch = fx.torch
    # one step: the whole set is one batch, accumulators at zero
    dw, drms = fx.dev(w), torch.zeros((2, ot.STRIDE), dtype=torch.float32, device='cuda')
    fx.core.train(fx.dx[:n].contiguous(), fx.y[:n], rows, dw, drms, epochs=1, batch_size=n)
    got = dw.cpu().numpy()
    for i, (H, a, r, s) in enumerate(specs):
        k = ot.row_size(F, H)
        row, rms = w[i].astype(np.float64), np.zeros(ot.STRIDE)
        order = ot.shuffle(s, 0, n)
        m = ot.masks(s, 0, order, F, 0.2)
        _, g64, _ = ot.loss_grad(row, F, H, fx.x[order], fx.y[order].astype(np.float64), m, 0.8, a, r)
        _, g32, _ = ot.loss_grad(row.astype(np.float32), F, H, fx.x[order].astype(np.float32), fx.y[order].astype(np.float32),
                                 m.astype(np.float32), 0.8, a, r, np.float32)
        spread = np.max(np.abs(g32 - g64))
        ot.rmsprop(row, rms, g64)
        clear = np.abs(g64[:k]) > 100 * spread
        assert clear.mean() > 0.5
        assert np.max(np.abs(got[i, :k][clear] - row[:k][clear])) < 1e-5
        assert not np.any(got[i, k:])
    # three epochs of batches of 16: the loss curve within 1e-3 (relative), 99 % of the weights within 1e-4 and all within
    # the largest change RMSprop can make in those steps
    dw, drms = fx.dev(w), torch.zeros((2, ot.STRIDE), dtype=torch.float32, device='cuda')
    loss = fx.core.train(fx.dx[:n].contiguous(), fx.y[:n], rows, dw, drms, epochs=3, batch_size=16).cpu().numpy()
    got = dw.cpu().numpy()
    for i, (H, a, r, s) in enumerate(specs):
        k = ot.row_size(F, H)
        row, rms = w[i].astype(np.float64), np.zeros(ot.STRIDE)
        want = ot.train_row(row, rms, F, H, fx.x, fx.y.astype(np.float64), np.arange(n), s, 3, batch_size=16,
                            activation=a, recurrent_activation=r)
        assert np.allclose(loss[i], want, rtol=1e-3), (loss[i], want)
        d = np.abs(got[i, :k] - row[:k])
        assert np.quantile(d, 0.99) < 1e-4 and d.max() < 12 * 2 * 0.001 / np.sqrt(0.1), (np.quantile(d, 0.99), d.max())


# ---- 4. determinism ---------------------------------------------------------------------------------------------------------

@gpu
def test_bit_for_bit_determinism(fx):
    torch = fx.torch
    specs = [(20, 'linear', 'hard_sigmoid', 1), (8, 'tanh', 'sigmoid', 2), (24, 'linear', 'sigmoid', 3)]
    rows, w = fx.rows(specs)

    def run(rows, w, epochs=3, epoch0=0, rms=None, pairs=None):
        dw = fx.dev(w)
        drms = torch.zeros_like(dw) if rms is None else rms
        kw = {} if pairs is None else dict(rows_of=pairs[0], recs=pairs[1])
        loss = fx.core.train(fx.dx, fx.y, rows, dw, drms, epochs=epochs, epoch0=epoch0, batch_size=37, **kw)
        return dw, drms, loss

    a = run(rows, w)
    b = run(rows, w)
    assert all(_same(x.cpu().numpy(), y.cpu().numpy()) for x, y in zip(a, b))
    # a row alone, and among the others in reverse order
    for i, sp in enumerate(specs):
        alone = run(fx.core.train_rows([sp[0]], [sp[1]], [sp[2]], [sp[3]]), w[i:i + 1])
        assert _same(alone[0].cpu().numpy()[0], a[0].cpu().numpy()[i])
        assert _same(alone[2].cpu().numpy()[0], a[2].cpu().numpy()[i])
    rev = specs[::-1]
    r = run(fx.core.train_rows(*[[s[c] for s in rev] for c in range(4)]), w[::-1].copy())
    assert _same(r[0].cpu().numpy()[::-1].copy(), a[0].cpu().numpy())
    # E epochs in one call equal E calls with epoch0 advancing
    dw = fx.dev(w)
    drms = torch.zeros_like(dw)
    losses = []
    for e in range(3):
        losses.append(fx.core.train(fx.dx, fx.y, rows, dw, drms, epochs=1, epoch0=e, batch_size=37))
    assert _same(dw.cpu().numpy(), a[0].cpu().numpy()) and _same(drms.cpu().numpy(), a[1].cpu().numpy())
    assert _same(torch.cat(losses, 1).cpu().numpy(), a[2].cpu().numpy())
    # pairs: a row with no entries is untouched and gets NaN losses
    pr = np.asarray([0] * 50 + [2] * 30, np.int32)
    pc = np.arange(80, dtype=np.int32)
    p = run(rows, w, pairs=(pr, pc))
    pw, pl = p[0].cpu().numpy(), p[2].cpu().numpy()
    assert _same(pw[1], w[1]) and np.all(np.isnan(pl[1])) and not np.any(np.isnan(pl[[0, 2]]))


# ---- 5. end to end ------------------------------------------------------------------------------------------------------------

@gpu
def test_training_lifts_test_pool_accuracy_and_pool_train_reloads(fx, tmp_path, capsys):
    m = fx.m
    torch = fx.torch
    clips, tg = train_task.dataset(0, train_task.N_TRAIN)
    t_clips, t_tg = train_task.dataset(10000, train_task.N_TEST)
    core = m.PreciseB200()
    core.set_pool(1)
    init = m.GruModel.init(13, 20, 0)
    core.pool_load(0, init)
    before = m.offline.test_pool(core, t_clips, t_tg, np.zeros(1, np.int32))[0].accuracy()
    state = m.offline.TrainState.from_models(core, [init], [0])
    inputs = m.offline.vectorize_clips(core, clips)
    loss, val = m.offline.train(core, state, inputs, tg, epochs=train_task.EPOCHS, batch_size=train_task.BATCH,
                                validation=(m.offline.vectorize_clips(core, t_clips), t_tg))
    assert state.epoch == train_task.EPOCHS and loss.shape == val.shape == (1, train_task.EPOCHS)
    trained = state.models()[0]
    core.pool_load(0, trained)
    after = m.offline.test_pool(core, t_clips, t_tg, np.zeros(1, np.int32))[0].accuracy()
    assert before < 0.7 and after >= train_task.MIN_ACCURACY, (before, after)
    assert val[0, -1] < val[0, 0]
    core.close()
    # pool_train: the slot's ticks score the returned weights, bit for bit as a fresh pool_load of them
    S, chunk = 4, 1024
    sb = m.StreamBatch(init, S)
    sb.set_pool(2)
    sb.pool_load(1, init)
    sb.set_stream_pool(np.full(S, 1, np.int32))
    out = sb.pool_train([1], [init], clips[:40], tg[:40], epochs=2, batch_size=16)
    ref = m.StreamBatch(init, S)
    ref.set_pool(2)
    ref.pool_load(1, out[0])
    ref.set_stream_pool(np.full(S, 1, np.int32))
    pcm = np.stack([np.resize(clips[i], 8 * chunk) for i in range(S)])
    for k in range(8):
        x = torch.from_numpy(pcm[:, k * chunk:(k + 1) * chunk].copy()).cuda()
        a, b = sb.update_pool(x), ref.update_pool(x)
        assert _same(a['raw'].cpu().numpy(), b['raw'].cpu().numpy())
    # the command line: two new models on a folder of wavs, then precise-test reads them
    d = tmp_path / 'data'
    for sub, cl, t in (('', clips[:40], tg[:40]), ('test', t_clips[:20], t_tg[:20])):
        for i, (c, y) in enumerate(zip(cl, t)):
            folder = d / sub / ('wake-word' if y else 'not-wake-word')
            folder.mkdir(parents=True, exist_ok=True)
            with wave.open(str(folder / ('c%03d.wav' % i)), 'wb') as w:
                w.setnchannels(1); w.setsampwidth(2); w.setframerate(16000); w.writeframes(c.tobytes())
    names = [str(tmp_path / 'a.npz'), str(tmp_path / 'b.npz')]
    from mycroft_precise_b200 import test as ptest
    from mycroft_precise_b200 import train as ptrain
    ptrain.main(names + [str(d), '-e', '2', '-b', '16'])
    text = capsys.readouterr().out
    assert text.count('Epoch 2/2 - loss: ') == 2 and 'val_loss' in text
    for n in names:
        assert os.path.isfile(n) and os.path.isfile(n + '.params')
    ptest.main(names + [str(d), '-nf'])
    text = capsys.readouterr().out
    assert text.count('.npz ===') == 2


# ---- 6. refusals ----------------------------------------------------------------------------------------------------------------

@gpu
def test_refused_calls_change_nothing(fx):
    m = fx.m
    torch = fx.torch
    lib = fx.core.lib
    h = fx.core._h
    rows, w = fx.rows([(20, 'linear', 'hard_sigmoid', 1), (8, 'tanh', 'sigmoid', 2)])
    arr, k = rows
    dw = fx.dev(w)
    drms = torch.full_like(dw, 0.5)
    dloss = torch.zeros((k, 2), dtype=torch.float64, device='cuda')
    w0, r0 = dw.cpu().numpy().copy(), drms.cpu().numpy().copy()
    tg = np.ascontiguousarray(fx.y)
    vp = lambda t: C.c_void_p(t.data_ptr())
    tp = tg.ctypes.data_as(C.c_void_p)
    pr = np.asarray([0, 1, 2], np.int32)
    pc = np.asarray([0, 1, 2], np.int32)
    pc_bad = np.asarray([0, 1, 400], np.int32)
    o = m.core.pb_train_opts()
    assert lib.pb_train_opts_default(C.byref(o)) == 0
    assert (o.epochs, o.epoch0, o.batch_size, o.loss_bias) == (10, 0, 5000, np.float32(0.8))

    def train(opts=o, **kw):
        a = dict(h=h, x=vp(fx.dx), n=400, tg=tp, rows=arr, k=k, pr=None, pc=None, np_=0, w=vp(dw), rms=vp(drms), loss=vp(dloss))
        a.update(kw)
        return lib.pb_train(a['h'], a['x'], a['n'], a['tg'], a['rows'], a['k'], a['pr'], a['pc'], a['np_'],
                            C.byref(opts) if opts is not None else None, a['w'], a['rms'], a['loss'], None)

    def opts(**kw):
        x = m.core.pb_train_opts()
        lib.pb_train_opts_default(C.byref(x))
        for key, v in kw.items():
            setattr(x, key, v)
        return x

    bad_row = (m.core.pb_train_row * 1)(m.core.pb_train_row(25, 0, 0, 0))
    bad_act = (m.core.pb_train_row * 1)(m.core.pb_train_row(20, 2, 0, 0))
    refusals = [dict(h=None), dict(opts=None), dict(x=None), dict(tg=None), dict(rows=None), dict(k=-1), dict(n=-1),
                dict(w=None), dict(rms=None), dict(rows=bad_row, k=1), dict(rows=bad_act, k=1),
                dict(pr=pr.ctypes.data_as(C.c_void_p), pc=None, np_=3), dict(pr=np.asarray([0, 1, 2], np.int32).ctypes.data_as(C.c_void_p),
                                                                         pc=pc.ctypes.data_as(C.c_void_p), np_=3),
                dict(pr=np.asarray([0, 1, 1], np.int32).ctypes.data_as(C.c_void_p), pc=pc_bad.ctypes.data_as(C.c_void_p), np_=3),
                dict(opts=opts(epochs=0)), dict(opts=opts(epoch0=-1)), dict(opts=opts(batch_size=0)),
                dict(opts=opts(lr=float('nan'))), dict(opts=opts(rho=1.0)), dict(opts=opts(epsilon=-1.0)),
                dict(opts=opts(loss_bias=1.5)), dict(opts=opts(dropout=1.0))]
    for kw in refusals:
        assert train(**kw) == -1, kw
    torch.cuda.synchronize()
    assert _same(dw.cpu().numpy(), w0) and _same(drms.cpu().numpy(), r0)
    # pb_train_loss's own refusals
    L = lambda **kw: lib.pb_train_loss(h, vp(fx.dx), 400, tp, arr, k, None, None, 0, kw.get('bias', 0.8), kw.get('rate', 0.0),
                                       kw.get('epoch', 0), vp(dw), kw.get('loss', vp(dloss)), None, None)
    assert L(epoch=-1) == -1 and L(loss=None) == -1 and L(bias=-0.1) == -1 and L(rate=1.0) == -1
    # pb_vectorize_clips: null output, empty clip; a handle with deltas is outside the fused front end
    pcm = fx.dev(_noise(4000, 1))
    out = torch.empty((2, T, F), dtype=torch.float32, device='cuda')
    assert lib.pb_vectorize_clips(h, vp(pcm), np.asarray([0, 2000, 4000], np.int64).ctypes.data_as(C.c_void_p), 2, 32767, 24000,
                                  None, None) == -1
    assert lib.pb_vectorize_clips(h, vp(pcm), np.asarray([0, 2000, 2000], np.int64).ctypes.data_as(C.c_void_p), 2, 32767, 24000,
                                  vp(out), None) == -1
    dcore = m.PreciseB200(m.ListenerParams(use_delta=True))
    with pytest.raises(NotImplementedError):
        dcore.vectorize_clips(pcm, np.asarray([0, 4000], np.int64))
    dx = torch.zeros((4, dcore.n_features, dcore.feature_size), dtype=torch.float32, device='cuda')
    with pytest.raises(NotImplementedError):
        dcore.train(dx, np.zeros(4, np.uint8), dcore.train_rows([20], ['linear'], ['hard_sigmoid'], [0]), fx.dev(w[:1]),
                    torch.zeros((1, ot.STRIDE), dtype=torch.float32, device='cuda'))
    dcore.close()
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
    rows, w = fx.rows([(20, 'linear', 'hard_sigmoid', 1)])
    x = core.vectorize_clips(fx.dev(_noise(30000, 2)), np.asarray([0, 30000], np.int64))
    core.train(x, np.ones(1, np.uint8), rows, fx.dev(w), torch.zeros((1, ot.STRIDE), dtype=torch.float32, device='cuda'), epochs=2)
    core.train_loss(x, np.ones(1, np.uint8), rows, fx.dev(w), grad=True)
    torch.cuda.synchronize()
    assert _same(core.export_streams(n=3).cpu().numpy(), before)
    assert np.array_equal(core.stream_pool(), ids)
    a = sb.update_pool(pcm)['raw'].cpu().numpy()
    ref = m.StreamBatch(g, 3)
    ref.set_pool(1)
    ref.pool_load(0, g)
    ref.set_stream_pool(np.zeros(3, np.int32))
    ref.update_pool(pcm)
    assert _same(ref.update_pool(pcm)['raw'].cpu().numpy(), a)
