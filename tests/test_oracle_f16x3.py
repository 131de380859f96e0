"""oracle.gru.gru_forward_f16x3, the reference for the fused family's fp16 x 3 scan, against the float64 GRU.  CPU only.

On small weights the split arithmetic must be as close to float64 as the float32 GRU is; on networks whose hidden state
leaves the fp16 range it must stay finite and make the float64 network's saturated decision (the kernel's split saturates
instead of overflowing to inf - inf = NaN)."""
import numpy as np
import pytest

from oracle import gru as og
from oracle.mfcc import vectorize_raw
from oracle.params import OracleParams


def windows(n=24, seed=0):
    """MFCC windows [n, 29, 13] of the oracle front end: noise from sigma 30 to 12 000, silence and half silence."""
    pr = OracleParams()
    rs = np.random.RandomState(seed)
    out = []
    for i in range(n):
        sigma = [30, 300, 3000, 12000][i % 4]
        a = np.clip(rs.randn(pr.buffer_samples) * sigma, -32768, 32767).astype(np.int16).astype(np.float32) / 32768
        if i % 6 == 4:
            a[:] = 0
        elif i % 6 == 5:
            a[:a.size // 2] = 0
        out.append(vectorize_raw(a, pr)[-pr.n_features:])
    return np.asarray(out, np.float32)


def doubling(H=20, F=13, sign=1.0):
    """z = 0, r = 1 and a recurrent candidate block of 2 I: h doubles every step (h_t = 2 h + 1), far past fp16's range."""
    kernel = np.zeros((F, 3 * H), np.float32)
    recurrent = np.zeros((H, 3 * H), np.float32)
    recurrent[:, 2 * H:] = 2 * np.eye(H)
    bias = np.concatenate([np.full(H, -10.0), np.full(H, 10.0), np.ones(H)])
    return og.GruWeights(kernel, recurrent, bias, np.full(H, sign * 0.1), 0.0)


def test_split_saturates():
    v = np.asarray([0.0, 1.0, -3.1415927, 65503.0, 65504.0, 65519.0, 65520.0, 1e6, -1e30, 6e-8], np.float32)
    hi, lo = og.split_f16(v)
    assert np.all(np.isfinite(hi)) and np.all(np.isfinite(lo))
    assert np.all(np.abs(hi) <= og.F16_MAX) and np.all(np.abs(lo) <= og.F16_MAX)
    small = np.abs(v) < og.F16_MAX
    assert np.all(np.abs((hi + lo)[small] - v[small]) <= 2.0 ** -22 * np.abs(v[small]) + 2.0 ** -24)
    assert np.array_equal(np.sign(hi + lo), np.sign(v))
    assert np.isinf(og.split_f16(np.float32(1e6), saturate=False)[0])


@pytest.mark.parametrize('act', [('linear', 'hard_sigmoid'), ('tanh', 'sigmoid'), ('linear', 'sigmoid'),
                                 ('tanh', 'hard_sigmoid')])
def test_small_weights_match_float64(act):
    """Within 1e-7 on noise.  Silent windows (every row c0 = -36) lose most to the 22-bit split of x: up to 2.1e-7."""
    x = windows()
    silent = np.arange(len(x)) % 6 == 4
    worst = np.zeros(2)
    for H in (1, 7, 16, 20, 24):
        w = og.GruWeights.random(13, H, seed=H, scale=0.1)
        w.activation, w.recurrent_activation = act
        p, lg = og.gru_forward_f16x3(w, x)
        p64, _ = og.gru_forward(w, x, np.float64)
        assert p.dtype == np.float32 and lg.dtype == np.float32
        e = np.abs(p - p64)
        worst = np.maximum(worst, [e[~silent].max(), e[silent].max()])
    print('%s / %s: max |p_f16x3 - p64| %.3g (noise), %.3g (silence)' % (act + tuple(worst)))
    assert worst[0] < 1e-7 and worst[1] < 3e-7


@pytest.mark.parametrize('sign', [1.0, -1.0])
@pytest.mark.parametrize('H', [16, 20])
def test_doubling_network_saturates(H, sign):
    x = windows(12, seed=H)
    w = doubling(H, sign=sign)
    _, _, h64 = og.gru_forward(w, x, np.float64, return_hidden=True)
    assert np.all(h64 > 1e8)                                         # far outside fp16
    p64, _ = og.gru_forward(w, x, np.float64)
    p, lg = og.gru_forward_f16x3(w, x)
    assert np.all(np.isfinite(p)) and np.all(np.isfinite(lg))
    want = 1.0 if sign > 0 else 0.0
    assert np.all(np.abs(p64 - want) < 1e-12)
    assert np.all(p == np.float32(want))
