"""oracle.gru.gru_forward_tf32x3, the reference for the wide networks' 3 x TF32 scan, against the float64 GRU.  CPU only.

The splits must reproduce their operands to TF32 x 2 precision and round the way the kernel and the host do; on small weights
the split arithmetic must be as close to float64 as the float32 GRU is; on networks whose hidden state doubles every step
(h near 2^T, inside float32's range for T <= 100) it must stay finite and make the float64 network's saturated decision."""
import numpy as np
import pytest

from oracle import gru as og
from oracle.mfcc import add_deltas, vectorize_raw
from oracle.params import OracleParams

ACTS = (('linear', 'hard_sigmoid'), ('tanh', 'sigmoid'), ('linear', 'sigmoid'), ('tanh', 'hard_sigmoid'))


def windows(n=24, seed=0, delta=False):
    """MFCC windows [n, 29, 13] (with deltas [n, 29, 26]) of the oracle front end: noise from sigma 30 to 12 000, silence and
    half silence."""
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
        v = vectorize_raw(a, pr)[-pr.n_features:]
        out.append(add_deltas(v) if delta else v)
    return np.asarray(out, np.float32)


def doubling(H, F, sign):
    """z = 0, r = 1 and a recurrent candidate block of 2 I: h_t = 2 h_(t-1) + 1 in every unit, whatever the input; the Dense
    layer, sign (1e-4 sum(h) / H - 2), saturates once h is past about 20 000."""
    recurrent = np.zeros((H, 3 * H), np.float32)
    recurrent[:, 2 * H:] = 2 * np.eye(H)
    bias = np.concatenate([np.full(H, -10.0), np.full(H, 10.0), np.ones(H)])
    return og.GruWeights(np.zeros((F, 3 * H)), recurrent, bias, np.full(H, 1e-4 * sign / H), -2.0 * sign)


def test_split_round_trip():
    """Weights (rounded halves): |hi + lo - v| <= 2^-22 |v|.  Operands (truncated halves, the lower one truncated again by
    the tensor core): < 2^-21 |v|.  hi and lo are TF32 numbers."""
    rs = np.random.RandomState(0)
    v = np.concatenate([rs.randn(20000) * 10.0 ** rs.uniform(-30, 30, 20000),
                        [1.0, -1.0, 3.1415927, 1e-30, 65504.0, 2.0 ** 100, -(2.0 ** 120) * 1.7]]).astype(np.float32)
    v64 = v.astype(np.float64)
    for split, bound in ((og.split_tf32_weights, 2.0 ** -22), (og.split_tf32, 2.0 ** -21)):
        hi, lo = split(v)
        err = np.abs(hi + lo - v64)
        assert np.all(err <= bound * np.abs(v64)), (split.__name__, float(np.max(err / np.abs(v64))))
        for part in (hi, lo):
            bits = part.astype(np.float32).view(np.uint32)
            assert np.all(bits & 0x1fff == 0)
    # the two roundings: a value half-way between TF32 neighbours goes up on the host, down in the kernel's hi
    half = np.float32(1 + 2.0 ** -11)
    assert og.split_tf32_weights(half)[0] == 1 + 2.0 ** -10 and og.split_tf32(half)[0] == 1.0
    assert og.split_tf32_weights(half)[1] == -(2.0 ** -11) and og.split_tf32(half)[1] == 2.0 ** -11


@pytest.mark.parametrize('act', ACTS)
@pytest.mark.parametrize('delta', [False, True])
def test_small_weights_match_float64(act, delta):
    """std 0.1 / sqrt(H / 20) weights, H from 1 to 128: max |p_tf32x3 - p64| within 2 max |p32 - p64| + 1e-7 on every
    network, and below 2e-7 overall."""
    x = windows(delta=delta)
    F = x.shape[2]
    worst = np.zeros(2)
    for H in (1, 7, 17, 24, 33, 64, 100, 128):
        w = og.GruWeights.random(F, H, seed=H, scale=0.1 / np.sqrt(max(H, 20) / 20.0))
        w.activation, w.recurrent_activation = act
        p, lg = og.gru_forward_tf32x3(w, x)
        assert p.dtype == np.float32 and lg.dtype == np.float32
        p64 = og.gru_forward(w, x, np.float64)[0]
        p32 = og.gru_forward(w, x, np.float32)[0].astype(np.float64)
        e, e32 = np.max(np.abs(p - p64)), np.max(np.abs(p32 - p64))
        assert e <= 2 * e32 + 1e-7, (H, e, e32)
        worst = np.maximum(worst, [e, e32])
    print('%s / %s, deltas %s: max |p_tf32x3 - p64| %.3g, max |p32 - p64| %.3g' % (act + (delta,) + tuple(worst)))
    assert worst[0] < 2e-7


@pytest.mark.parametrize('sign', [1.0, -1.0])
@pytest.mark.parametrize('H,F,T', [(20, 13, 29), (7, 26, 29), (33, 40, 73), (128, 13, 100)])
def test_doubling_network_decides(H, F, T, sign):
    """h reaches 2^T - 1 (2^100 at T = 100, inside float32): finite, and exactly the float64 network's decision."""
    x = (np.random.RandomState(H + T).randn(6, T, F) * 10).astype(np.float32)
    w = doubling(H, F, sign)
    with np.errstate(over='ignore'):                               # exp(-logit) of the saturated decision
        p64, _, h64 = og.gru_forward(w, x, np.float64, return_hidden=True)
    assert np.all(h64 == 2.0 ** T - 1)
    want = 1.0 if sign > 0 else 0.0
    assert np.all(np.abs(p64 - want) < 1e-12)
    p, lg = og.gru_forward_tf32x3(w, x)
    assert np.all(np.isfinite(lg)) and np.all(np.sign(lg) == sign)
    assert np.all(p == np.float32(want))
