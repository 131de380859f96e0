"""oracle/train.py at pb_train_wide's row stride: the same float64 restatement of training (GRU with reset_after = False,
Dense(1, sigmoid), the weighted log loss, per-gate input dropout, RMSprop), for rows of WIDE_STRIDE floats and up to 128 GRU
units.  oracle/train.py's loss_grad returns rows of its fixed STRIDE (2 980 floats, 24 units at most), so the gradient's
BPTT is restated here with the row width as an argument; keys, masks, shuffles, activations, the row layout and RMSprop are
oracle/train.py's own functions.  With stride=ot.STRIDE the results equal oracle/train.py's (tests/test_train_wide_host.py).
TEST INFRASTRUCTURE ONLY."""
import numpy as np

from oracle import train as ot

WIDE_STRIDE = 55812                 # PB_TRAIN_WIDE_STRIDE: 3 H (F + H + 1) + H + 1 = 55 809 at H = 128, F = 16, rounded up


def pack(model, stride=WIDE_STRIDE):
    """A GruModel-like object -> float32 row [stride] (ot.pack's layout)."""
    flat = np.concatenate([np.asarray(model.kernel, np.float32).ravel(), np.asarray(model.recurrent, np.float32).ravel(),
                           np.asarray(model.bias, np.float32).ravel(), np.asarray(model.dense_w, np.float32).ravel(),
                           np.asarray([model.dense_b], np.float32)])
    out = np.zeros(stride, np.float32)
    out[:flat.size] = flat
    return out


def loss_grad(row, F, H, x, y, mask, loss_bias, activation='linear', recurrent_activation='hard_sigmoid', dtype=np.float64,
              kink=0.0, stride=WIDE_STRIDE):
    """ot.loss_grad with a gradient row of ``stride`` floats: (loss, gradient [stride], sum of the per-entry losses)."""
    dt = np.dtype(dtype).type
    w = ot.unpack(np.asarray(row, dtype), F, H)
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
        z, dz_da = ot._act(recurrent_activation, az, dt, kink)
        r, dr_da = ot._act(recurrent_activation, ar, dt, kink)
        ah = xm[:, 2, t] @ K[:, 2 * H:] + b[2 * H:] + (r * h) @ U[:, 2 * H:]
        hh, dhh_da = ot._act(activation, ah, dt)
        saved.append((h, z, r, hh, dz_da, dr_da, dhh_da))
        h = z * h + (dt(1) - z) * hh
    logit = h @ dw + dw.dtype.type(db)
    p = dt(1) / (dt(1) + np.exp(-logit))
    lb = dt(loss_bias)
    per = lb * (-(dt(1) - y) * np.log(dt(1) - p + dt(ot.EPS))) + (dt(1) - lb) * (-y * np.log(p + dt(ot.EPS)))
    loss = per.sum() / dt(B)
    dp = (lb * (dt(1) - y) / (dt(1) - p + dt(ot.EPS)) - (dt(1) - lb) * y / (p + dt(ot.EPS))) / dt(B)
    dlogit = dp * p * (dt(1) - p)
    gK, gU, gb = np.zeros_like(K), np.zeros_like(U), np.zeros_like(b)
    gdw = h.T @ dlogit
    gdb = dlogit.sum()
    dh = dlogit[:, None] * dw[None, :]
    for t in range(T - 1, -1, -1):
        hp, z, r, hh, dz_da, dr_da, dhh_da = saved[t]
        daz = dh * (hp - hh) * dz_da
        dah = dh * (dt(1) - z) * dhh_da
        drh = dah @ U[:, 2 * H:].T
        dar = drh * hp * dr_da
        dh = dh * z + drh * r + daz @ U[:, :H].T + dar @ U[:, H:2 * H].T
        gU[:, :H] += hp.T @ daz
        gU[:, H:2 * H] += hp.T @ dar
        gU[:, 2 * H:] += (r * hp).T @ dah
        gK[:, :H] += xm[:, 0, t].T @ daz
        gK[:, H:2 * H] += xm[:, 1, t].T @ dar
        gK[:, 2 * H:] += xm[:, 2, t].T @ dah
        gb[:H] += daz.sum(0)
        gb[H:2 * H] += dar.sum(0)
        gb[2 * H:] += dah.sum(0)
    g = np.zeros(stride, dtype)
    flat = np.concatenate([gK.ravel(), gU.ravel(), gb, gdw, [gdb]])
    g[:flat.size] = flat
    return loss, g, per.sum()


def train_row(row, rms, F, H, inputs, targets, recs, seed, epochs, epoch0=0, batch_size=5000, lr=0.001, rho=0.9,
              eps=ot.EPS, loss_bias=0.8, dropout=0.2, activation='linear', recurrent_activation='hard_sigmoid',
              dtype=np.float64, stride=WIDE_STRIDE):
    """ot.train_row (pb_train_wide for one row) on rows of ``stride`` floats: row and rms float64 [stride], updated in place.
    Returns the epoch losses."""
    n = len(recs)
    recs = np.asarray(recs, np.int64)
    losses = []
    for e in range(epoch0, epoch0 + epochs):
        order = ot.shuffle(seed, e, n)
        tot = 0.0
        for b0 in range(0, n, batch_size):
            js = order[b0:b0 + batch_size]
            m = ot.masks(seed, e, js, F, dropout)
            _, g, s = loss_grad(row, F, H, inputs[recs[js]], targets[recs[js]], m, loss_bias, activation,
                                recurrent_activation, dtype, stride=stride)
            tot += float(s)
            ot.rmsprop(row, rms, g.astype(np.float64), lr, rho, eps)
        losses.append(tot / n)
    return losses
