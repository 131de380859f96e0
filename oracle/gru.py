"""Oracle restatement of the network forward pass.  TEST INFRASTRUCTURE ONLY.  ** PARITY UNPINNED **

The network is defined by the reference at ``precise/model.py:77-82``::

    Sequential([GRU(recurrent_units, activation='linear', input_shape=(n_features, feature_size),
                    dropout=..., name='net'),
                Dense(1, activation='sigmoid')])

and evaluated by ``KerasRunner.predict`` / ``TensorFlowRunner.predict``
(``precise/network_runner.py:88-92`` / ``:69-71``) -- both stateless: every call starts from
h0 = 0 and scans all ``n_features`` rows (``Listener.update``, ``network_runner.py:148-153``).

The arithmetic lives in Keras (<=2.1.5 per ``setup.py:78``; 2.2.4 per ``requirements.txt:11``)
on TensorFlow 1.13 CPU, neither of which is present.  Published Keras GRU semantics restated:

  * weights ``kernel[F, 3H]``, ``recurrent_kernel[H, 3H]``, ``bias[3H]``; gate order z, r, h
  * recurrent_activation = hard_sigmoid(x) = clip(0.2 x + 0.5, 0, 1)   (Keras default)
  * reset_after = False (Keras default): the reset gate multiplies h BEFORE the matmul
        z  = hs(x Wz + h Uz + bz)
        r  = hs(x Wr + h Ur + br)
        hh = act(x Wh + (r * h) Uh + bh)      act = linear here (model.py:78)
        h' = z * h + (1 - z) * hh
  * return_sequences = False, dropout inactive at inference
  * Dense: y = sigmoid(h_T Wd + bd);   Keras casts inputs to float32.

``activation`` / ``recurrent_activation`` are parameters because a saved model's config may
override them (the weight importer reads them).
"""
import numpy as np


def hard_sigmoid(x):
    return np.clip(0.2 * x + 0.5, 0.0, 1.0)


def sigmoid(x):
    one = x.dtype.type(1)
    return one / (one + np.exp(-x))


_ACT = {
    'linear': lambda x: x,
    'tanh': np.tanh,
    'hard_sigmoid': hard_sigmoid,
    'sigmoid': sigmoid,
}


class GruWeights:
    """Plain container: kernel[F,3H], recurrent[H,3H], bias[3H], dense_w[H], dense_b."""

    def __init__(self, kernel, recurrent, bias, dense_w, dense_b,
                 activation='linear', recurrent_activation='hard_sigmoid'):
        self.kernel = np.ascontiguousarray(kernel, dtype=np.float32)
        self.recurrent = np.ascontiguousarray(recurrent, dtype=np.float32)
        self.bias = np.ascontiguousarray(bias, dtype=np.float32).reshape(-1)
        self.dense_w = np.ascontiguousarray(dense_w, dtype=np.float32).reshape(-1)
        self.dense_b = float(np.float32(np.asarray(dense_b).reshape(-1)[0]))
        self.activation = activation
        self.recurrent_activation = recurrent_activation
        self.F = self.kernel.shape[0]
        self.H = self.recurrent.shape[0]
        assert self.kernel.shape == (self.F, 3 * self.H)
        assert self.recurrent.shape == (self.H, 3 * self.H)
        assert self.bias.shape == (3 * self.H,)
        assert self.dense_w.shape == (self.H,)

    @staticmethod
    def random(F=13, H=20, seed=0, scale=0.3):
        """Seeded synthetic weights (no trained model ships with the reference)."""
        rs = np.random.RandomState(seed)
        return GruWeights(rs.randn(F, 3 * H) * scale, rs.randn(H, 3 * H) * scale,
                          rs.randn(3 * H) * scale, rs.randn(H) * scale, rs.randn(1) * scale)


def gru_forward(w: GruWeights, x: np.ndarray, dtype=np.float32, return_hidden=False):
    """x[N, T, F] -> (prob[N], logit[N]) in ``dtype``.  Batched over N; sequential over T."""
    x = np.asarray(x).astype(dtype)
    if x.ndim == 2:
        x = x[None]
    N, T, F = x.shape
    assert F == w.F, (F, w.F)
    H = w.H
    K = w.kernel.astype(dtype)
    U = w.recurrent.astype(dtype)
    b = w.bias.astype(dtype)
    act = _ACT[w.activation]
    ract = _ACT[w.recurrent_activation]
    h = np.zeros((N, H), dtype=dtype)
    for t in range(T):
        a = x[:, t, :] @ K + b                       # input projection, all three gates
        zr = ract(a[:, :2 * H] + h @ U[:, :2 * H])
        z, r = zr[:, :H], zr[:, H:]
        hh = act(a[:, 2 * H:] + (r * h) @ U[:, 2 * H:])
        h = z * h + (dtype(1) - z) * hh
    logit = h @ w.dense_w.astype(dtype) + dtype(w.dense_b)
    prob = sigmoid(logit)
    if return_hidden:
        return prob, logit, h
    return prob, logit


F16_MAX = 65504.0


def _f16(v, saturate):
    """float32 v rounded to the nearest fp16 (as float32); ``saturate``: +-65504 instead of +-inf for |v| >= 65520."""
    with np.errstate(over='ignore'):
        h = np.asarray(v, np.float32).astype(np.float16).astype(np.float32)
    if saturate:
        h = np.where(np.isinf(h) & np.isfinite(v), np.copysign(np.float32(F16_MAX), v), h).astype(np.float32)
    return h


def split_f16(v, saturate=True):
    """float32 v -> (hi, lo), float64 values of fp16 numbers: hi = fp16(v), lo = fp16(v - hi) with v - hi in float32.
    ``saturate``: the kernel's operand split (cvt.rn.satfinite); otherwise the host's weight split (build_frag16)."""
    v = np.asarray(v, np.float32)
    hi = _f16(v, saturate)
    with np.errstate(invalid='ignore'):
        lo = _f16(v - hi, saturate)
    return hi.astype(np.float64), lo.astype(np.float64)


def _mm3(a, b):
    """a . b as the fused family's fp16 x 3 products: a_lo b_hi + a_hi b_lo + a_hi b_hi (lo . lo dropped), summed in
    float64.  a: (hi, lo) of a split operand, b: (hi, lo) of a split weight matrix."""
    with np.errstate(invalid='ignore'):
        return a[1] @ b[0] + a[0] @ b[1] + a[0] @ b[0]


def _f32(v):
    return np.asarray(v, np.float64).astype(np.float32)


_ACT32 = {
    'linear': lambda x: x,
    'tanh': lambda x: np.tanh(x.astype(np.float32)),
    'hard_sigmoid': lambda x: np.clip(_f32(np.float64(np.float32(0.2)) * x.astype(np.float64) + 0.5), 0, 1),
    'sigmoid': lambda x: sigmoid(x.astype(np.float32)),
}


def gru_forward_f16x3(w: GruWeights, x: np.ndarray):
    """x[N, T, F] -> (prob[N], logit[N]) float32, as the fused family's tensor-core scan (gru_bank.cuh: bank_scan) computes
    them: every product x . W, h . U and (r * h) . U in fp16 x 3 with operands split by ``split_f16`` (saturating, as the
    kernel splits x, h and r * h) and weights by the host's non-saturating split.  Each product is summed exactly and added
    to the float32 accumulator in the kernel's order: bias, then the x part, then the h part.  Activations are float32
    (hard_sigmoid as fma(0.2, x, 0.5)), r * h is rounded to float32 before its split, h = fma(z, h, (1 - z) a) is rounded to
    float32 and the Dense layer is summed exactly and rounded once.  A reference for tests: what the scan should return,
    not a model of the tensor cores' internal rounding."""
    x = np.asarray(x, np.float32)
    if x.ndim == 2:
        x = x[None]
    N, T, F = x.shape
    assert F == w.F, (F, w.F)
    H = w.H
    K = split_f16(w.kernel, saturate=False)
    Uzr = split_f16(w.recurrent[:, :2 * H], saturate=False)
    Uh = split_f16(w.recurrent[:, 2 * H:], saturate=False)
    b = w.bias.astype(np.float64)
    act, ract = _ACT32[w.activation], _ACT32[w.recurrent_activation]
    h = np.zeros((N, H), np.float32)
    for t in range(T):
        ax = _f32(b + _mm3(split_f16(x[:, t, :]), K))                 # bias, then the x part
        zr = ract(_f32(ax[:, :2 * H].astype(np.float64) + _mm3(split_f16(h), Uzr)))
        z, r = zr[:, :H].astype(np.float32), zr[:, H:].astype(np.float32)
        rh = _f32(r.astype(np.float64) * h)
        a = act(_f32(ax[:, 2 * H:].astype(np.float64) + _mm3(split_f16(rh), Uh))).astype(np.float32)
        p = _f32((np.float32(1) - z).astype(np.float64) * a)
        h = _f32(z.astype(np.float64) * h + p)
    logit = _f32(h.astype(np.float64) @ w.dense_w.astype(np.float64) + w.dense_b)
    return sigmoid(logit), logit


_TF32_MASK = np.uint32(0xffffe000)


def _tf32_trunc(v):
    """float32 v with its 13 low mantissa bits cleared (float32)."""
    return (np.asarray(v, np.float32).view(np.uint32) & _TF32_MASK).view(np.float32)


def _tf32_round(v):
    """float32 v rounded to TF32 as the host's weight split does: (bits + 0x1000) & 0xffffe000 (float32)."""
    u = np.asarray(v, np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & _TF32_MASK).view(np.float32)


def split_tf32_weights(v):
    """float32 weights v -> (hi, lo) as upload_wide splits them: hi = v rounded to TF32, lo = (v - hi) rounded to TF32, with
    v - hi in float32.  float64 values."""
    v = np.asarray(v, np.float32)
    hi = _tf32_round(v)
    lo = _tf32_round(v - hi)
    return hi.astype(np.float64), lo.astype(np.float64)


def split_tf32(v):
    """float32 operands v -> (hi, lo) as gru_wide_kernel splits x, h and r * h (split_tf32 in gru_kernels.cuh): hi = v with
    the 13 low mantissa bits cleared, lo = v - hi in float32 (exact).  The tensor core then reads only lo's top 19 bits;
    that truncation is an assumption about the hardware (the PTX ISA leaves a .tf32 operand's unused bits unspecified), and
    lo is returned truncated so.  float64 values; |hi + lo - v| < 2^-21 |v|."""
    v = np.asarray(v, np.float32)
    hi = _tf32_trunc(v)
    lo = _tf32_trunc(v - hi)
    return hi.astype(np.float64), lo.astype(np.float64)


def gru_forward_tf32x3(w: GruWeights, x: np.ndarray):
    """x[N, T, F] -> (prob[N], logit[N]) float32, as the wide networks' tensor-core scan (gru_wide.cuh: gru_wide_kernel, 3 x
    TF32) computes them: each gate's pre-activation is the bias plus the products lo . hi + hi . lo + hi . hi (lo . lo
    dropped) of operands split by ``split_tf32`` and weights split by ``split_tf32_weights``, summed exactly and rounded to
    float32 once.  z and r come from one product over [x | h], the candidate from one over [x | r * h].  Activations are
    float32 (hard_sigmoid as fma(0.2, x, 0.5)), r * h is rounded to float32 before its split, h = fma(z, h, (1 - z) a) is
    rounded to float32 and the Dense layer is an fmaf chain from the bias over the units in order.  A reference for tests:
    what the scan should return, not a model of the tensor cores' internal rounding."""
    x = np.asarray(x, np.float32)
    if x.ndim == 2:
        x = x[None]
    N, T, F = x.shape
    assert F == w.F, (F, w.F)
    H = w.H
    Kzr, Kh = split_tf32_weights(w.kernel[:, :2 * H]), split_tf32_weights(w.kernel[:, 2 * H:])
    Uzr, Uh = split_tf32_weights(w.recurrent[:, :2 * H]), split_tf32_weights(w.recurrent[:, 2 * H:])
    b = w.bias.astype(np.float64)
    act, ract = _ACT32[w.activation], _ACT32[w.recurrent_activation]
    h = np.zeros((N, H), np.float32)
    with np.errstate(over='ignore', invalid='ignore'):
        for t in range(T):
            xs = split_tf32(x[:, t, :])
            zr = ract(_f32(b[:2 * H] + _mm3(xs, Kzr) + _mm3(split_tf32(h), Uzr)))
            z, r = zr[:, :H].astype(np.float32), zr[:, H:].astype(np.float32)
            rh = _f32(r.astype(np.float64) * h)
            a = act(_f32(b[2 * H:] + _mm3(xs, Kh) + _mm3(split_tf32(rh), Uh))).astype(np.float32)
            p = _f32((np.float32(1) - z).astype(np.float64) * a)
            h = _f32(z.astype(np.float64) * h + p)
        logit = np.full(N, np.float32(w.dense_b), np.float32)
        for j in range(H):
            logit = _f32(h[:, j].astype(np.float64) * np.float64(w.dense_w[j]) + logit)
        return sigmoid(logit), logit


def predict(w: GruWeights, inputs: np.ndarray) -> np.ndarray:
    """``Runner.predict`` contract (network_runner.py:35-37): [N,T,F] -> float32 [N,1]."""
    return gru_forward(w, inputs, np.float32)[0].astype(np.float32)[:, None]


def run(w: GruWeights, inp: np.ndarray) -> float:
    """``Runner.run`` contract (network_runner.py:73-74 / :94-95): [T,F] -> scalar."""
    return predict(w, inp[np.newaxis])[0][0]
