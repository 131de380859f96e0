"""Training without a device: the float64 restatement of pb_train (oracle/train.py) against torch.autograd and central
finite differences, fixed values of its key, mask and shuffle functions, the weight-row packing against GruModel, and the
synthetic task the GPU tests train on (tests/train_task.py)."""
import os
import sys

import numpy as np
import pytest

from oracle import train as ot

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import train_task  # noqa: E402

PAIRS = [('linear', 'hard_sigmoid'), ('tanh', 'sigmoid'), ('linear', 'sigmoid'), ('tanh', 'hard_sigmoid')]


def _row(F, H, seed, scale=0.5):
    rs = np.random.RandomState(seed)
    row = np.zeros(ot.STRIDE)
    row[:ot.row_size(F, H)] = rs.randn(ot.row_size(F, H)) * scale
    return row


def _torch_loss(row, F, H, x, y, mask, bias, act, ract):
    import torch
    w = torch.tensor(row[:ot.row_size(F, H)], dtype=torch.float64, requires_grad=True)
    a = 0
    parts = []
    for n in (F * 3 * H, H * 3 * H, 3 * H, H, 1):
        parts.append(w[a:a + n])
        a += n
    K, U, b, dw, db = parts[0].view(F, 3 * H), parts[1].view(H, 3 * H), parts[2], parts[3], parts[4]
    fa = {'linear': lambda v: v, 'tanh': torch.tanh}[act]
    fr = {'sigmoid': torch.sigmoid, 'hard_sigmoid': lambda v: torch.clamp(0.2 * v + 0.5, 0, 1)}[ract]
    x = torch.tensor(x)
    m = torch.tensor(mask)
    yt = torch.tensor(y)
    h = torch.zeros(x.shape[0], H, dtype=torch.float64)
    for t in range(x.shape[1]):
        xz, xr, xh = x[:, t] * m[:, 0], x[:, t] * m[:, 1], x[:, t] * m[:, 2]
        z = fr(xz @ K[:, :H] + b[:H] + h @ U[:, :H])
        r = fr(xr @ K[:, H:2 * H] + b[H:2 * H] + h @ U[:, H:2 * H])
        hh = fa(xh @ K[:, 2 * H:] + b[2 * H:] + (r * h) @ U[:, 2 * H:])
        h = z * h + (1 - z) * hh
    p = torch.sigmoid(h @ dw + db)
    loss = bias * torch.mean(-(1 - yt) * torch.log(1 - p + 1e-7)) + (1 - bias) * torch.mean(-yt * torch.log(p + 1e-7))
    loss.backward()
    return loss.item(), w.grad.detach().numpy()


@pytest.mark.parametrize('act,ract', PAIRS)
@pytest.mark.parametrize('H', [1, 8, 20, 24])
@pytest.mark.parametrize('rate', [0.0, 0.3])
def test_gradient_equals_autograd(act, ract, H, rate):
    pytest.importorskip('torch')
    F, T, B = 13, 9, 6
    rs = np.random.RandomState(H)
    x = rs.randn(B, T, F)
    y = (rs.rand(B) < 0.5).astype(np.float64)
    m = ot.masks(7, 3, range(B), F, rate)
    row = _row(F, H, H + 1)
    loss, g, _ = ot.loss_grad(row, F, H, x, y, m, 0.8, act, ract)
    tl, tg = _torch_loss(row, F, H, x, y, m, 0.8, act, ract)
    n = ot.row_size(F, H)
    assert abs(loss - tl) <= 1e-12 * max(1.0, abs(tl))
    assert np.max(np.abs(g[:n] - tg)) <= 1e-10 * max(1.0, np.max(np.abs(tg)))
    assert not np.any(g[n:])


@pytest.mark.parametrize('act,ract', PAIRS)
@pytest.mark.parametrize('label', [0, 1, None])
def test_gradient_equals_finite_differences(act, ract, label):
    """Central differences in float64, including batches with one label only."""
    F, H, T, B = 5, 4, 6, 7
    rs = np.random.RandomState(11)
    x = rs.randn(B, T, F)
    y = (rs.rand(B) < 0.5).astype(np.float64) if label is None else np.full(B, float(label))
    m = ot.masks(1, 0, range(B), F, 0.3)
    row = _row(F, H, 12)
    _, g, _ = ot.loss_grad(row, F, H, x, y, m, 0.7, act, ract)
    n = ot.row_size(F, H)
    fd = np.zeros(n)
    for i in range(n):
        rp, rm = row.copy(), row.copy()
        rp[i] += 1e-6
        rm[i] -= 1e-6
        fd[i] = (ot.loss_grad(rp, F, H, x, y, m, 0.7, act, ract)[0] - ot.loss_grad(rm, F, H, x, y, m, 0.7, act, ract)[0]) / 2e-6
    assert np.max(np.abs(fd - g[:n])) < 1e-7


def test_key_mask_and_shuffle_known_values():
    assert ot.mix(0) == 0
    assert ot.key(1, 2, 3, 4) == 18275852912223555758
    assert ot.key(1, 2, 3, 4) == ot.mix(ot.mix(ot.mix(ot.mix(1) + 2) + 3) + 4)
    assert list(ot.shuffle(7, 0, 10)) == [2, 9, 4, 1, 6, 5, 7, 8, 3, 0]
    assert list(ot.shuffle(7, 1, 10)) != list(ot.shuffle(7, 0, 10))
    k = ot.keep(3, 5, 17, 13, 0.2)
    assert k.shape == (3, 13) and 0.6 < k.mean() < 0.95
    assert np.all(ot.keep(3, 5, 17, 13, 0.0))
    m = ot.masks(3, 5, [17], 13, 0.2)
    assert set(np.unique(m)) <= {0.0, np.float64(np.float32(1) / np.float32(0.8))}
    # the mask is a fixed function of (seed, epoch, entry)
    assert np.array_equal(ot.keep(3, 5, 17, 13, 0.2), k)


def test_row_packing_round_trips_with_gru_model():
    from mycroft_precise_b200.model_io import GruModel
    for H in (1, 20, 24):
        m = GruModel.random(16, H, seed=H)
        row = ot.pack(m)
        assert row.shape == (ot.STRIDE,) and not np.any(row[ot.row_size(16, H):])
        w = ot.unpack(row, 16, H)
        assert np.array_equal(w['kernel'], m.kernel) and np.array_equal(w['recurrent'], m.recurrent)
        assert np.array_equal(w['bias'], m.bias) and np.array_equal(w['dense_w'], m.dense_w)
        assert float(w['dense_b']) == np.float32(m.dense_b)
    assert ot.row_size(16, 24) == 2977 <= ot.STRIDE


def test_gru_model_init_follows_keras_initialisers():
    from mycroft_precise_b200.model_io import GruModel
    m = GruModel.init(13, 20, seed=3)
    assert np.abs(m.kernel).max() <= np.sqrt(6 / (13 + 60)) and np.abs(m.dense_w).max() <= np.sqrt(6 / 21)
    assert np.allclose(m.recurrent @ m.recurrent.T, np.eye(20), atol=1e-5)        # orthonormal rows
    assert not np.any(m.bias) and m.dense_b == 0
    assert np.array_equal(GruModel.init(13, 20, seed=3).kernel, m.kernel)


def test_oracle_training_learns_the_synthetic_task():
    """The rehearsal of the GPU end-to-end test: accuracy on held-out clips from about chance to MIN_ACCURACY."""
    from mycroft_precise_b200.model_io import GruModel
    from oracle import mfcc as om
    from oracle.gru import GruWeights, gru_forward
    from oracle.params import OracleParams
    opr = OracleParams()
    clips, y = train_task.dataset(0, train_task.N_TRAIN)
    t_clips, t_y = train_task.dataset(10000, train_task.N_TEST)
    X = np.stack([om.vectorize(c.astype(np.float64) / 32767.0, opr) for c in clips])
    tX = np.stack([om.vectorize(c.astype(np.float64) / 32767.0, opr) for c in t_clips])

    def accuracy(row):
        w = ot.unpack(row, 13, 20)
        p = gru_forward(GruWeights(w['kernel'], w['recurrent'], w['bias'], w['dense_w'], w['dense_b']), tX, np.float64)[0]
        return np.mean((p > 0.5) == (t_y > 0))

    row = ot.pack(GruModel.init(13, 20, 0)).astype(np.float64)
    rms = np.zeros_like(row)
    before = accuracy(row)
    losses = ot.train_row(row, rms, 13, 20, X, y.astype(np.float64), np.arange(len(clips)), seed=0, epochs=train_task.EPOCHS,
                          batch_size=train_task.BATCH, dropout=0.2)
    after = accuracy(row)
    assert before < 0.7 and after >= train_task.MIN_ACCURACY, (before, after)
    assert losses[-1] < losses[0]


def _fma32(a, x, b):
    """float32 fmaf(a, x, b): the product of two float32 values and the sum with b are exact in float64 here (|a x| < 1,
    b = 0.5), so one rounding to float32 is the fused result."""
    return np.float32(np.float64(np.float32(a)) * np.float64(np.float32(x)) + np.float64(np.float32(b)))


def test_hard_sigmoid_gradient_bounds_and_why_the_kernel_does_not_fuse():
    """hard_sigmoid's gradient is 0.2 where 0 <= 0.2 x + 0.5 <= 1, bounds included, with 0.2 x rounded before + 0.5 (Keras's
    float32 order).  At x = -2.5 that is 0 exactly in float64 and float32, so both include it; fmaf rounds once and gives
    -2^-27, which would exclude it.  Just past +2.5 float32 rounds 1 + 2^-24 to 1 (a tie to even) and includes the point
    where float64 does not: an inherent float32 difference that the restatement shares with the kernel."""
    f32 = np.float32
    lo, hi = f32(-2.5), f32(2.5)
    below, above = np.nextafter(lo, f32(-np.inf)), np.nextafter(hi, f32(np.inf))
    inside = [np.nextafter(lo, f32(0)), lo, f32(0), hi, np.nextafter(hi, f32(0))]
    for dt in (np.float64, np.float32):
        for x in inside:
            y, g = ot._act('hard_sigmoid', np.asarray([x], dt), dt)
            assert g[0] == dt(0.2) and 0 <= y[0] <= 1, (dt, x)
        assert ot._act('hard_sigmoid', np.asarray([below], dt), dt)[1][0] == 0
        y, _ = ot._act('hard_sigmoid', np.asarray([lo, hi], dt), dt)
        assert y[0] == 0 and y[1] == 1
    # float64 excludes the float just past 2.5; float32's mul-then-add includes it
    assert ot._act('hard_sigmoid', np.asarray([above], np.float64), np.float64)[1][0] == 0
    assert ot._act('hard_sigmoid', np.asarray([above], np.float32), np.float32)[1][0] == f32(0.2)
    # the fused form moves the lower bound: -2.5 falls out, and nothing else of these points changes side
    s = _fma32(0.2, lo, 0.5)
    assert s == -f32(2.0 ** -27) and s < 0
    assert f32(0.2) * lo + f32(0.5) == 0
    for x in [below, above] + inside:
        if x != lo:
            assert (0 <= _fma32(0.2, x, 0.5) <= 1) == (0 <= f32(0.2) * x + f32(0.5) <= 1), x
    assert _fma32(0.2, hi, 0.5) == 1


@pytest.mark.parametrize('seed,epoch', [(0, 0), (1, 5), (2 ** 31, 2 ** 31 - 1), (2 ** 32 - 1, 5), (2 ** 32 - 1, 2 ** 31 - 1)])
def test_mask_counter_layout_up_to_47(seed, epoch):
    """keep's [g, f] is counter 1 + c of the key with c = 3 f + g, c up to 47 at F = 16: the device reads c < 32 from one
    ballot over counters 1 + lane and c >= 32 from a second over 33 + lane.  A smaller F keeps F = 16's first F columns."""
    rate = np.float32(0.5)
    for j in (0, 1, 70):
        base = ot.mix(ot.mix(ot.mix(seed) + epoch) + j)
        assert all(ot.key(seed, epoch, j, c) == ot.mix(base + c) for c in (0, 1, 33, 48))
        u = lambda c: np.float32(float(ot.mix(base + c) >> 40) * 2.0 ** -24)
        m0 = sum(1 << lane for lane in range(32) if u(1 + lane) >= rate)
        m1 = sum(1 << lane for lane in range(32) if u(33 + lane) >= rate)
        mask = m0 | (m1 << 32)
        k = ot.keep(seed, epoch, j, 16, rate)
        for f in range(16):
            for g in range(3):
                assert bool((mask >> (3 * f + g)) & 1) == k[g, f], (j, f, g)
        assert 8 < np.count_nonzero(~k) < 40            # rate 0.5: a fair share of the 48 columns dropped
        for F in (1, 5, 13):
            assert np.array_equal(ot.keep(seed, epoch, j, F, rate), k[:, :F])
