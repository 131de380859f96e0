"""Training of the fused-family network, restated in numpy: what pb_train and pb_train_loss compute on the device.
TEST INFRASTRUCTURE ONLY.  ** KERAS PARITY UNPINNED **

The reference trains with Keras ``fit`` (precise/model.py:57-91, scripts/train.py:159-166): the GRU of oracle/gru.py,
``Dense(1, sigmoid)``, the loss of precise/functions.py:39-50 with ``loss_bias = 1 - sensitivity`` (train.py:86), input
dropout of the Keras 2.1/2.2 GRU (implementation 1: three masks per entry, one per gate z, r, h, each [feature_size],
fixed over the time steps, kept elements scaled by 1 / (1 - rate); no recurrent dropout) and RMSprop at Keras's defaults.
Randomness is defined rather than drawn, so that the device can reproduce it bit for bit:

  mix              the splitmix64 finalizer
  key(s, e, j, c)  mix(mix(mix(mix(s) + e) + j) + c) on uint64 (s the row's seed, e the epoch, j the entry's index within
                   its row in request order)
  shuffle          a row's entries sorted ascending by (key(s, e, j, 0), j)
  dropout          feature f of gate g is kept iff float32((key(s, e, j, 1 + 3 f + g) >> 40) 2^-24) >= rate

A weight row is Keras's order, flat: kernel[F][3H], recurrent[H][3H], bias[3H], dense_w[H], dense_b, then zeros up to
STRIDE floats.
"""
import numpy as np

STRIDE = 2980                       # PB_TRAIN_STRIDE: 3 H (F + H + 1) + H + 1 = 2977 at H = 24, F = 16, rounded up
M64 = (1 << 64) - 1
EPS = 1e-7                          # Keras's epsilon: the loss's log floor and RMSprop's


def mix(z):
    """splitmix64's finalizer on a Python int (uint64 wraparound)."""
    z &= M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def key(s, e, j, c):
    return mix(mix(mix(mix(s) + e) + j) + c)


def shuffle(seed, epoch, n):
    """The order in which a row's n entries (indices j in request order) are visited in ``epoch``."""
    return np.asarray(sorted(range(n), key=lambda j: (key(seed, epoch, j, 0), j)), np.int64)


def keep(seed, epoch, j, F, rate):
    """[3, F] bool: whether input feature f reaches gate g (0, 1, 2 = z, r, h) for entry j in ``epoch``."""
    out = np.zeros((3, F), bool)
    for f in range(F):
        for g in range(3):
            u = np.float32(float(key(seed, epoch, j, 1 + 3 * f + g) >> 40) * 2.0 ** -24)
            out[g, f] = u >= np.float32(rate)
    return out


def masks(seed, epoch, js, F, rate):
    """[n, 3, F] float64 input masks of entries js: 1 / (1 - rate) in float32 where kept, else 0; all ones at rate 0."""
    scale = np.float64(np.float32(1.0) / (np.float32(1.0) - np.float32(rate)))
    return np.stack([keep(seed, epoch, int(j), F, rate) * scale for j in js]) if len(js) else np.zeros((0, 3, F))


def row_size(F, H):
    return 3 * H * (F + H + 1) + H + 1


def pack(model):
    """A GruModel-like object (kernel, recurrent, bias, dense_w, dense_b) -> float32 row [STRIDE]."""
    parts = [np.asarray(model.kernel, np.float32).ravel(), np.asarray(model.recurrent, np.float32).ravel(),
             np.asarray(model.bias, np.float32).ravel(), np.asarray(model.dense_w, np.float32).ravel(),
             np.asarray([model.dense_b], np.float32)]
    flat = np.concatenate(parts)
    out = np.zeros(STRIDE, np.float32)
    out[:flat.size] = flat
    return out


def unpack(row, F, H):
    """Row -> dict(kernel [F, 3H], recurrent [H, 3H], bias [3H], dense_w [H], dense_b) views of the row's dtype."""
    row = np.asarray(row)
    a = 0
    out = {}
    for name, shape in (('kernel', (F, 3 * H)), ('recurrent', (H, 3 * H)), ('bias', (3 * H,)), ('dense_w', (H,)),
                        ('dense_b', ())):
        n = int(np.prod(shape)) if shape else 1
        out[name] = row[a:a + n].reshape(shape) if shape else row[a]
        a += n
    return out


def _act(name, x, dt):
    if name == 'linear':
        return x, np.ones_like(x)
    if name == 'tanh':
        y = np.tanh(x)
        return y, dt(1) - y * y
    if name == 'sigmoid':
        y = dt(1) / (dt(1) + np.exp(-x))
        return y, y * (dt(1) - y)
    if name == 'hard_sigmoid':
        s = dt(0.2) * x + dt(0.5)
        return np.clip(s, 0, 1), np.where((s >= 0) & (s <= 1), dt(0.2), dt(0))
    raise ValueError(name)


def loss_grad(row, F, H, x, y, mask, loss_bias, activation='linear', recurrent_activation='hard_sigmoid', dtype=np.float64):
    """One batch: x [B, T, F], y [B] (0 / 1), mask [B, 3, F] (masks()).  Returns (loss, gradient row [STRIDE], sum of the
    per-entry losses): loss = bias mean(-(1-y) log(1-p+1e-7)) + (1-bias) mean(-y log(p+1e-7)) and its gradient by
    hand-written BPTT, everything in ``dtype``."""
    dt = np.dtype(dtype).type
    w = unpack(np.asarray(row, dtype), F, H)
    K, U, b, dw, db = w['kernel'], w['recurrent'], w['bias'], w['dense_w'], w['dense_b']
    x = np.asarray(x, dtype)
    y = np.asarray(y, dtype)
    B, T, _ = x.shape
    xm = x[:, None, :, :] * np.asarray(mask, dtype)[:, :, None, :]     # [B, 3, T, F]: the input each gate sees
    h = np.zeros((B, H), dtype)
    saved = []
    for t in range(T):
        az = xm[:, 0, t] @ K[:, :H] + b[:H] + h @ U[:, :H]
        ar = xm[:, 1, t] @ K[:, H:2 * H] + b[H:2 * H] + h @ U[:, H:2 * H]
        z, dz_da = _act(recurrent_activation, az, dt)
        r, dr_da = _act(recurrent_activation, ar, dt)
        ah = xm[:, 2, t] @ K[:, 2 * H:] + b[2 * H:] + (r * h) @ U[:, 2 * H:]
        hh, dhh_da = _act(activation, ah, dt)
        saved.append((h, z, r, hh, dz_da, dr_da, dhh_da))
        h = z * h + (dt(1) - z) * hh
    logit = h @ dw + dw.dtype.type(db)
    p = dt(1) / (dt(1) + np.exp(-logit))
    lb = dt(loss_bias)
    per = lb * (-(dt(1) - y) * np.log(dt(1) - p + dt(EPS))) + (dt(1) - lb) * (-y * np.log(p + dt(EPS)))
    loss = per.sum() / dt(B)
    dp = (lb * (dt(1) - y) / (dt(1) - p + dt(EPS)) - (dt(1) - lb) * y / (p + dt(EPS))) / dt(B)
    dlogit = dp * p * (dt(1) - p)
    gK, gU, gb = np.zeros_like(K), np.zeros_like(U), np.zeros_like(b)
    gdw = h.T @ dlogit
    gdb = dlogit.sum()
    dh = dlogit[:, None] * dw[None, :]
    for t in range(T - 1, -1, -1):
        hp, z, r, hh, dz_da, dr_da, dhh_da = saved[t]
        daz = dh * (hp - hh) * dz_da
        dah = dh * (dt(1) - z) * dhh_da
        dhp = dh * z
        drh = dah @ U[:, 2 * H:].T
        dar = drh * hp * dr_da
        dhp = dhp + drh * r + daz @ U[:, :H].T + dar @ U[:, H:2 * H].T
        gU[:, :H] += hp.T @ daz
        gU[:, H:2 * H] += hp.T @ dar
        gU[:, 2 * H:] += (r * hp).T @ dah
        gK[:, :H] += xm[:, 0, t].T @ daz
        gK[:, H:2 * H] += xm[:, 1, t].T @ dar
        gK[:, 2 * H:] += xm[:, 2, t].T @ dah
        gb[:H] += daz.sum(0)
        gb[H:2 * H] += dar.sum(0)
        gb[2 * H:] += dah.sum(0)
        dh = dhp
    g = np.zeros(STRIDE, dtype)
    flat = np.concatenate([gK.ravel(), gU.ravel(), gb, gdw, [gdb]])
    g[:flat.size] = flat
    return loss, g, per.sum()


def rmsprop(w, a, g, lr=0.001, rho=0.9, eps=EPS):
    """Keras's RMSprop step in place: a = rho a + (1 - rho) g^2; w -= lr g / (sqrt(a) + eps)."""
    a *= rho
    a += (1 - rho) * g * g
    w -= lr * g / (np.sqrt(a) + eps)


def train_row(row, rms, F, H, inputs, targets, recs, seed, epochs, epoch0=0, batch_size=5000, lr=0.001, rho=0.9,
              eps=EPS, loss_bias=0.8, dropout=0.2, activation='linear', recurrent_activation='hard_sigmoid',
              dtype=np.float64):
    """pb_train for one row in ``dtype``: row and rms are float64 arrays [STRIDE] updated in place, recs the row's clips in
    request order (entry j is clip recs[j]).  Returns the epoch losses (the batch-size-weighted mean of the batch losses)."""
    n = len(recs)
    recs = np.asarray(recs, np.int64)
    losses = []
    for e in range(epoch0, epoch0 + epochs):
        order = shuffle(seed, e, n)
        tot = 0.0
        for b0 in range(0, n, batch_size):
            js = order[b0:b0 + batch_size]
            m = masks(seed, e, js, F, dropout)
            _, g, s = loss_grad(row, F, H, inputs[recs[js]], targets[recs[js]], m, loss_bias, activation,
                                recurrent_activation, dtype)
            tot += float(s)
            g = g.astype(np.float64)
            rmsprop(row, rms, g, lr, rho, eps)
        losses.append(tot / n)
    return losses
