"""The training oracle at pb_train_wide's stride (tests/train_wide_oracle.py), without a device: its gradient against
torch.autograd in float64 and against central differences for 25 to 128 GRU units, equality with oracle/train.py at the
fused stride, the row packing at both strides, and the fused stride left as it was."""
import os
import sys

import numpy as np
import pytest

from oracle import train as ot

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import train_wide_oracle as wo  # noqa: E402
from test_train_host import PAIRS, _torch_loss  # noqa: E402

WS = wo.WIDE_STRIDE


def _row(F, H, seed, scale=0.3):
    rs = np.random.RandomState(seed)
    row = np.zeros(WS)
    row[:ot.row_size(F, H)] = rs.randn(ot.row_size(F, H)) * scale / np.sqrt(H / 8)
    return row


def test_strides():
    assert ot.STRIDE == 2980
    assert ot.row_size(16, 128) == 55809 and WS == 55812 and WS % 4 == 0
    from mycroft_precise_b200.core import PB_TRAIN_STRIDE, PB_TRAIN_WIDE_STRIDE
    assert (PB_TRAIN_STRIDE, PB_TRAIN_WIDE_STRIDE) == (ot.STRIDE, WS)
    text = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'include', 'precise_b200.h')).read()
    assert '#define PB_TRAIN_STRIDE 2980' in text and '#define PB_TRAIN_WIDE_STRIDE 55812' in text


@pytest.mark.parametrize('act,ract', PAIRS)
@pytest.mark.parametrize('H', [25, 32, 64, 120, 128])
@pytest.mark.parametrize('rate', [0.0, 0.3])
def test_gradient_equals_autograd(act, ract, H, rate):
    pytest.importorskip('torch')
    F, T, B = 13, 5, 4
    rs = np.random.RandomState(H)
    x = rs.randn(B, T, F)
    y = (np.arange(B) % 2).astype(np.float64)
    mask = ot.masks(H, 2, range(B), F, rate)
    row = _row(F, H, H + 1)
    loss, g, s = wo.loss_grad(row, F, H, x, y, mask, 0.8, act, ract)
    assert g.shape == (WS,) and not np.any(g[ot.row_size(F, H):])
    tl, tg = _torch_loss(row, F, H, x, y, mask, 0.8, act, ract)
    n = ot.row_size(F, H)
    assert abs(loss - tl) <= 1e-12 * max(1.0, abs(tl)) and abs(s / B - loss) <= 1e-12
    assert np.allclose(g[:n], tg, rtol=1e-9, atol=1e-12), np.max(np.abs(g[:n] - tg))


@pytest.mark.parametrize('act,ract', [('tanh', 'sigmoid'), ('linear', 'sigmoid')])
@pytest.mark.parametrize('H', [25, 64, 128])
def test_gradient_equals_finite_differences(act, ract, H):
    F, T, B = 5, 4, 3
    rs = np.random.RandomState(7 + H)
    x = rs.randn(B, T, F)
    y = np.asarray([1.0, 0.0, 1.0])
    mask = ot.masks(3, 0, range(B), F, 0.3)
    row = _row(F, H, H)
    _, g, _ = wo.loss_grad(row, F, H, x, y, mask, 0.7, act, ract)
    n = ot.row_size(F, H)
    idx = np.random.RandomState(H).choice(n, 60, replace=False)
    idx = np.concatenate([idx, [0, 3 * H * F, 3 * H * (F + H), n - 1]])             # first of each block and dense_b
    eps = 1e-6
    for i in idx:
        a, b = row.copy(), row.copy()
        a[i] += eps
        b[i] -= eps
        fd = (wo.loss_grad(a, F, H, x, y, mask, 0.7, act, ract)[0]
              - wo.loss_grad(b, F, H, x, y, mask, 0.7, act, ract)[0]) / (2 * eps)
        assert abs(fd - g[i]) <= 1e-6 * max(1.0, abs(g[i])), (i, fd, g[i])


@pytest.mark.parametrize('H', [1, 20, 24, 25, 64, 128])
def test_row_packing_round_trips_at_both_strides(H):
    from mycroft_precise_b200.model_io import GruModel
    m = GruModel.random(16, H, seed=H, scale=0.2)
    for stride in ((ot.STRIDE, WS) if H <= 24 else (WS,)):
        row = wo.pack(m, stride)
        assert row.shape == (stride,) and row.dtype == np.float32 and not np.any(row[ot.row_size(16, H):])
        u = ot.unpack(row, 16, H)
        for name in ('kernel', 'recurrent', 'bias', 'dense_w'):
            assert np.array_equal(u[name], getattr(m, name)), name
        assert u['dense_b'] == np.float32(m.dense_b)
    if H <= 24:
        assert np.array_equal(wo.pack(m)[:ot.STRIDE], ot.pack(m)) and np.array_equal(wo.pack(m, ot.STRIDE), ot.pack(m))


@pytest.mark.parametrize('act,ract', PAIRS)
@pytest.mark.parametrize('dtype', [np.float64, np.float32])
def test_restatement_is_oracle_train_at_the_fused_stride(act, ract, dtype):
    F, H, B = 13, 24, 5
    rs = np.random.RandomState(3)
    x = rs.randn(B, 7, F)
    y = (np.arange(B) % 2).astype(np.float64)
    mask = ot.masks(9, 1, range(B), F, 0.4)
    row = _row(F, H, 4)[:ot.STRIDE]
    for kink in (0.0, 2e-5):
        a = ot.loss_grad(row, F, H, x, y, mask, 0.8, act, ract, dtype, kink)
        b = wo.loss_grad(row, F, H, x, y, mask, 0.8, act, ract, dtype, kink, stride=ot.STRIDE)
        assert a[0] == b[0] and a[2] == b[2] and a[1].dtype == b[1].dtype and np.array_equal(a[1], b[1])


def test_train_row_at_the_wide_stride_is_the_fused_one_padded():
    F, H = 13, 8
    rs = np.random.RandomState(0)
    x = rs.randn(20, 3, F)
    y = (np.arange(20) % 2).astype(np.float64)
    a = _row(F, H, 1)
    b = a[:ot.STRIDE].copy()
    ra, rb = np.zeros(WS), np.zeros(ot.STRIDE)
    la = wo.train_row(a, ra, F, H, x, y, np.arange(20), 5, 2, batch_size=6)
    lb = ot.train_row(b, rb, F, H, x, y, np.arange(20), 5, 2, batch_size=6)
    assert la == lb and np.array_equal(a[:ot.STRIDE], b) and not np.any(a[ot.STRIDE:]) and np.array_equal(ra[:ot.STRIDE], rb)


def test_train_state_picks_its_layout_from_the_networks():
    pytest.importorskip('torch')
    from mycroft_precise_b200.model_io import GruModel
    from mycroft_precise_b200.offline import TrainState
    import torch

    class Core:                               # the parts of PreciseB200 from_models reads, on the CPU
        feature_size, device = 13, 'cpu'
        train_rows = staticmethod(lambda *a: (None, len(a[0])))
    Core.torch = torch
    narrow = [GruModel.init(13, 20, 0), GruModel.init(13, 24, 1)]
    wide = narrow + [GruModel.init(13, 25, 2)]
    a = TrainState.from_models(Core, narrow, [0, 1])
    b = TrainState.from_models(Core, wide, [0, 1, 2])
    assert not a.wide and a.stride == ot.STRIDE and tuple(a.weights.shape) == (2, ot.STRIDE)
    assert b.wide and b.stride == WS and tuple(b.weights.shape) == (3, WS)
    for st, models in ((a, narrow), (b, wide)):
        for got, m in zip(st.models(), models):
            assert got.hidden == m.hidden and np.array_equal(got.recurrent, m.recurrent) and np.array_equal(got.kernel, m.kernel)
