"""Training on the device (pb_vectorize_clips, pb_train, pb_train_loss) against the float64 restatement oracle/train.py over
every front end, hidden size, batch layout and optimizer setting the kernels accept.

- Front ends: feature sizes 1, 5, 13, 16 and 16 log-mels, and T = 1, 3, 19, 29, 73 and 112 steps (112 is the most the
  gradient kernel's shared memory holds: 231 632 of 232 448 bytes).  On each: the input rows of a mix of clips against the
  float64 vectorize, and one pb_train_loss call over forty rows (every hidden size of HIDDEN with every activation pair,
  1 to 129 entries per row, so tiles are partial and warps idle) at dropout 0 and 0.5 for three weight families.
- Gradients are compared block by block (kernel, recurrent and bias of each gate z / r / h, dense_w, dense_b): per block
  max |g_dev - g64| <= 10 max |g32 - g64| + 1e-6 max |g64|, with g64 and g32 loss_grad in float64 and float32; 1e-5 for a
  block of one element, and hard_sigmoid's jump added where a pre-activation lies within 1e-4 of a bound (check_grad;
  DESIGN.md section 6 "Training accuracy" has the measured errors).  A block that is all zero in float64 must be exactly
  zero on the device; every output must be finite.
- The dropout mask's (feature, gate) layout up to column 47, the shuffle order, RMSprop's arguments, the loss bias, a
  saturated Dense layer, the padding columns past a row's size and offline.train's path.
- hard_sigmoid's gradient at its bounds x = -2.5 and 2.5, which the kernel computes as Keras does (0.2 x rounded, then
  + 0.5; a fused multiply-add drops the lower bound).
- Calls split into several workspace groups, and the refused front ends and row sizes.

-m gpu throughout.  The per-block errors are printed (pytest -s) as "sweep:" lines."""
import numpy as np
import pytest

from oracle import mfcc as om
from oracle import train as ot
from oracle.params import OracleParams

gpu = pytest.mark.gpu
STRIDE = ot.STRIDE
HIDDEN = (1, 2, 3, 7, 8, 15, 16, 17, 23, 24)
ACTS = (('linear', 'hard_sigmoid'), ('tanh', 'sigmoid'), ('linear', 'sigmoid'), ('tanh', 'hard_sigmoid'))
COUNTS = (1, 3, 4, 5, 63, 64, 65, 129)          # entries per row: partial tiles, one tile, idle warps
SENTINEL = np.float32(-1234.5)                   # the padding columns' value; no call may change it
WS_CAP = 256 << 20                               # the training arena's per-group cap (TRAIN_WS_CAP in csrc/api.cu)
TILE = 64

FRONT_ENDS = {                 # name: ListenerParams arguments
    'default': {},                                      # F 13, T 29
    'f16': dict(n_mfcc=16),
    'f5': dict(n_mfcc=5, n_filt=12),
    'f1': dict(n_mfcc=1),
    'mels16': dict(vectorizer=1, n_filt=16, n_mfcc=16),
    't1': dict(buffer_t=0.1),
    't3': dict(buffer_t=0.2),
    't19': dict(buffer_t=1.0),
    't73': dict(hop_t=0.02, window_t=0.05),
    't112': dict(buffer_t=5.65),                        # the largest T the gradient kernel's shared memory holds
}
FAMILIES = ('std 0.1', 'keras init', 'tanh/sigmoid gain 2')
BLOCKS = tuple('%s %s' % (p, g) for p in ('kernel', 'recurrent', 'bias') for g in 'zrh') + ('dense_w', 'dense_b')


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


class Fixture:
    def __init__(self):
        import torch
        import mycroft_precise_b200 as m
        self.m, self.torch = m, torch
        self.cores = {}

    def core(self, name):
        if name not in self.cores:
            self.cores[name] = self.m.PreciseB200(self.m.ListenerParams(**FRONT_ENDS[name]))
        return self.cores[name]

    def dev(self, a):
        return self.torch.from_numpy(np.ascontiguousarray(a)).cuda()

    def close(self):
        for c in self.cores.values():
            c.close()


@pytest.fixture(scope='module')
def fx():
    pytest.importorskip('torch')
    f = Fixture()
    yield f
    f.close()


def _clips(max_samples, window, seed):
    """Noise at sigma 30 / 300 / 3000 / 12 000, silence, +32767, -32768 and a full-scale square wave, each at lengths 1,
    one window less one sample, exactly max_samples and above it."""
    rs = np.random.RandomState(seed)
    out = []
    for n in (1, window - 1, max_samples, max_samples + 777):
        for kind in range(8):
            if kind < 4:
                c = np.clip(rs.randn(n) * (30, 300, 3000, 12000)[kind], -32768, 32767)
            elif kind == 4:
                c = np.zeros(n)
            elif kind == 5:
                c = np.full(n, 32767)
            elif kind == 6:
                c = np.full(n, -32768)
            else:
                c = np.where((np.arange(n) // 37) % 2, 32767, -32767)
            out.append(c.astype(np.int16))
    return out


def _pack(clips):
    offsets = np.concatenate([[0], np.cumsum([len(c) for c in clips])]).astype(np.int64)
    return np.concatenate(clips), offsets


def _model(family, F, H, act, seed):
    m = __import__('mycroft_precise_b200').GruModel
    if family == 'std 0.1':
        return m.random(F, H, seed=seed, scale=0.1), act
    if family == 'keras init':
        return m.init(F, H, seed), act
    g = m.init(F, H, seed)
    return m(2 * g.kernel, 2 * g.recurrent, g.bias, 2 * g.dense_w, 0.0), ACTS[1]


def _blocks(g, F, H):
    w = ot.unpack(np.asarray(g, np.float64), F, H)
    out = {}
    for i, gate in enumerate('zrh'):
        out['kernel ' + gate] = w['kernel'][:, i * H:(i + 1) * H]
        out['recurrent ' + gate] = w['recurrent'][:, i * H:(i + 1) * H]
        out['bias ' + gate] = w['bias'][i * H:(i + 1) * H]
    out['dense_w'] = w['dense_w']
    out['dense_b'] = np.asarray([w['dense_b']])
    return out


KINK = 2e-5          # a band of 1e-4 in x around hard_sigmoid's bounds +-2.5 (2e-5 in s = 0.2 x + 0.5)


def check_grad(dev, g64, g32, F, H, what, jump=None, bad=None):
    """The per-block rule: max |g_dev - g64| <= 10 max |g32 - g64| + 1e-6 max |g64|, with 1e-5 for a block of one element
    (its float32 spread is a single sample and can be small by chance), plus, where hard_sigmoid's derivative jumps, the
    block's max |g_wide - g_narrow| (``jump``: float64 gradients with the 0.2 band widened and narrowed by KINK; nonzero only
    where a pre-activation lies within 1e-4 of a bound, so a float32 computation may fall on either side).  A block that is
    all zero in float64 (and in both bands) is exactly zero on the device.  Returns {block: (err, spread, max |g64|)};
    violations are appended to ``bad`` when it is given, else asserted."""
    n = ot.row_size(F, H)
    assert np.all(np.isfinite(dev)), what
    assert not np.any(dev[n:]), what
    d, a, b = _blocks(dev, F, H), _blocks(g64, F, H), _blocks(g32, F, H)
    jw, jn = (_blocks(jump[0], F, H), _blocks(jump[1], F, H)) if jump is not None else (a, a)
    out, fails = {}, []
    for name in BLOCKS:
        slack = float(np.max(np.abs(jw[name] - jn[name])))
        if not np.any(a[name]) and slack == 0:
            if np.any(d[name]):
                fails.append((what, name, 'not zero', float(np.max(np.abs(d[name])))))
            continue
        err = float(np.max(np.abs(d[name] - a[name])))
        spread = float(np.max(np.abs(b[name] - a[name])))
        top = float(np.max(np.abs(a[name])))
        bound = 10 * spread + (1e-6 if a[name].size > 1 else 1e-5) * top + slack
        if not err <= bound:
            fails.append((what, name, err, spread, top, slack, bound))
        out[name] = (err, spread, top)
    if bad is None:
        assert not fails, fails
    else:
        bad += fails
    return out


def check_loss(dev, l64, l32, what):
    assert np.isfinite(dev), what
    assert abs(dev - l64) <= 10 * abs(float(l32) - l64) + 1e-6 * abs(l64), (what, dev, l64, float(l32))


class Masks:
    """ot.masks, cached: the same (seed, epoch, rate) rows serve every family."""

    def __init__(self):
        self.c = {}

    def __call__(self, seed, epoch, n, F, rate):
        k = (seed, epoch, n, F, float(rate))
        if k not in self.c:
            self.c[k] = ot.masks(seed, epoch, range(n), F, rate)
        return self.c[k]


def oracle(specs, w, x, y, recs_of, F, rate, epoch, bias, masks, dtype, kink=0.0):
    out = []
    for i, (H, a, r, s) in enumerate(specs):
        recs = recs_of[i]
        m = masks(s, epoch, len(recs), F, rate)
        out.append(ot.loss_grad(w[i].astype(dtype), F, H, x[recs].astype(dtype), y[recs].astype(dtype), m.astype(dtype), bias,
                                a, r, dtype, kink)[:2] if kink == 0 or r == 'hard_sigmoid' else None)
    return out


def jumps(specs, w, x, y, recs_of, F, rate, epoch, bias, masks):
    """Per row (g_wide, g_narrow) in float64 for hard_sigmoid rows, None for sigmoid ones."""
    wide = oracle(specs, w, x, y, recs_of, F, rate, epoch, bias, masks, np.float64, KINK)
    narrow = oracle(specs, w, x, y, recs_of, F, rate, epoch, bias, masks, np.float64, -KINK)
    return [None if p is None else (p[1], q[1]) for p, q in zip(wide, narrow)]


def rows_of(counts, n_rec, seed):
    pr = np.concatenate([np.full(c, i, np.int32) for i, c in enumerate(counts)])
    pc = np.random.RandomState(seed).randint(0, n_rec, pr.size).astype(np.int32)
    return pr, pc, [pc[pr == i] for i in range(len(counts))]


def padded(w, specs, F):
    w = np.array(w, np.float32)
    for i, sp in enumerate(specs):
        w[i, ot.row_size(F, sp[0]):] = SENTINEL
    return w


def pad_ok(a, specs, F):
    return all(np.all(a[i, ot.row_size(F, sp[0]):] == SENTINEL) for i, sp in enumerate(specs))


# ---- 1. front ends ---------------------------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize('front', list(FRONT_ENDS))
def test_front_end_grid(fx, front):
    m = fx.m
    core = fx.core(front)
    pr = core.params
    F, T = core.feature_size, core.n_features
    assert (F, T) == (pr.feature_size, pr.n_features)
    if front == 't112':
        assert (T, pr.max_samples) == (112, 90400)
    # the input rows: the float64 vectorize and, bit for bit, the window score_dataset scores
    clips = _clips(pr.max_samples, pr.window_samples, 7)
    pcm, offsets = _pack(clips)
    dpcm = fx.dev(pcm)
    inputs = core.vectorize_clips(dpcm, offsets)
    got = inputs.cpu().numpy()
    assert got.shape == (len(clips), T, F) and np.all(np.isfinite(got))
    opr = OracleParams(**pr.to_dict())
    for j, c in enumerate(clips):
        if j % 8 in (5, 6) and len(c) >= pr.window_samples:
            # full-scale DC: the empty bands hold float32 FFT round-off, far above float64's floor, so the float64
            # vectorize is no yardstick there; these rows are checked through the scored window below
            continue
        want = om.vectorize(c.astype(np.float64) / 32767.0, opr)[..., :F]
        assert np.allclose(got[j], want, rtol=1e-4, atol=1e-3), (front, j, len(c), np.max(np.abs(got[j] - want)))
    if F == 13:
        # pb_predict's tensor-core scan of the default network is the pool's scan only for H 20, F 13
        g = m.GruModel.random(F, 20, seed=4, scale=0.1)
        core.load_weights(g.kernel, g.recurrent, g.bias, g.dense_w, g.dense_b)
        core.set_pool(1)
        core.pool_load(0, g)
        raw = core.score_dataset(dpcm, offsets, np.ones(len(clips), np.uint8), np.zeros(1, np.int32))['raw'].cpu().numpy()[0]
        core.gru_mode(2)
        try:
            assert _same(core.predict(inputs).cpu().numpy().reshape(-1), raw), front
        finally:
            core.gru_mode(0)
            core.set_pool(0)
    # forty rows, 1 .. 129 entries each, over the vectorized clips and as many random inputs
    x = np.concatenate([got, np.random.RandomState(1).randn(32, T, F).astype(np.float32) * 3])
    y = (np.random.RandomState(2).rand(len(x)) < 0.4).astype(np.uint8)
    dx = fx.dev(x)
    specs0 = [(H, a, r) for (a, r) in ACTS for H in HIDDEN]
    counts = [COUNTS[i % len(COUNTS)] for i in range(len(specs0))]
    pr_, pc_, recs_of = rows_of(counts, len(x), 3)
    masks = Masks()
    bad = []
    for family in FAMILIES:
        models = [_model(family, F, H, (a, r), 50 + i) for i, (H, a, r) in enumerate(specs0)]
        specs = [(H, act[0], act[1], 900 + i) for i, ((H, _a, _r), (_g, act)) in enumerate(zip(specs0, models))]
        w = padded(np.stack([ot.pack(mo) for mo, _ in models]), specs, F)
        dw = fx.dev(w)
        rows = core.train_rows(*[[s[c] for s in specs] for c in range(4)])
        for rate in (0.0, 0.5):
            loss, grad = core.train_loss(dx, y, rows, dw, pr_, pc_, loss_bias=0.8, dropout=rate, epoch=3, grad=True)
            loss, grad = loss.cpu().numpy(), grad.cpu().numpy()
            want = oracle(specs, w, x, y, recs_of, F, rate, 3, 0.8, masks, np.float64)
            f32 = oracle(specs, w, x, y, recs_of, F, rate, 3, 0.8, masks, np.float32)
            jump = jumps(specs, w, x, y, recs_of, F, rate, 3, 0.8, masks)
            worst = {}
            kinks = 0
            for i, (H, a, r, s) in enumerate(specs):
                what = (front, family, rate, H, a, r, counts[i])
                check_loss(loss[i], want[i][0], f32[i][0], what)
                kinks += jump[i] is not None and np.any(jump[i][0] != jump[i][1])
                for name, (err, spread, top) in check_grad(grad[i], want[i][1], f32[i][1], F, H, what, jump[i], bad).items():
                    e, q, rel = worst.get(name, (0.0, 0.0, 0.0))
                    worst[name] = (max(e, err), max(q, err / spread if spread > 0 else 0.0), max(rel, err / top))
            assert pad_ok(dw.cpu().numpy(), specs, F)
            print('sweep: %s | %s | dropout %.1f | worst |g_dev - g64| %.2g (%s) | worst ratio to |g32 - g64| %.3g (%s) | '
                  'worst |g_dev - g64| / max |g64| %.2g (%s) | rows with a gate within 1e-4 of +-2.5: %d'
                  % (front, family, rate, max(v[0] for v in worst.values()), max(worst, key=lambda k: worst[k][0]),
                     max(v[1] for v in worst.values()), max(worst, key=lambda k: worst[k][1]),
                     max(v[2] for v in worst.values()), max(worst, key=lambda k: worst[k][2]), kinks))
    assert not bad, bad


# ---- 2. the dropout mask's layout -------------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize('epoch', [0, 5, 2 ** 31 - 1])
def test_mask_layout_at_sixteen_features(fx, epoch):
    """F = 16, dropout 0.5, sigmoid gates (no gate gradient vanishes): the kernel-gradient columns of (feature, gate) that
    are exactly zero are those ot.keep drops, all 48 of them, for seeds 0, 1, 2^31 and 2^32 - 1.  The probe entry sits at
    j = 0, 5 and 70 of its row (the others have all-zero inputs, which add nothing to the kernel gradient), so the mask's
    entry index is checked in a second tile as well."""
    core = fx.core('f16')
    F, T = 16, core.n_features
    rs = np.random.RandomState(epoch % 97)
    probes = rs.randn(4, T, F).astype(np.float32)
    x = np.concatenate([np.zeros((1, T, F), np.float32), probes])
    y = np.asarray([0, 1, 0, 1, 1], np.uint8)
    specs, pr, pc, probe_j = [], [], [], []
    for si, seed in enumerate((0, 1, 2 ** 31, 2 ** 32 - 1)):
        for j in (0, 5, 70):
            i = len(specs)
            specs.append((8, ('linear', 'tanh')[i % 2], 'sigmoid', seed))
            pr += [i] * (j + 1)
            pc += [0] * j + [1 + si]
            probe_j.append(j)
    w = padded(np.random.RandomState(5).randn(len(specs), STRIDE) * 0.3, specs, F)
    dw = fx.dev(w)
    rows = core.train_rows(*[[s[c] for s in specs] for c in range(4)])
    pr, pc = np.asarray(pr, np.int32), np.asarray(pc, np.int32)
    _, grad = core.train_loss(fx.dev(x), y, rows, dw, pr, pc, loss_bias=0.8, dropout=0.5, epoch=epoch, grad=True)
    grad = grad.cpu().numpy()
    masks = Masks()
    recs_of = [pc[pr == i] for i in range(len(specs))]
    want = oracle(specs, w, x, y, recs_of, F, 0.5, epoch, 0.8, masks, np.float64)
    f32 = oracle(specs, w, x, y, recs_of, F, 0.5, epoch, 0.8, masks, np.float32)
    for i, (H, _a, _r, seed) in enumerate(specs):
        keep = ot.keep(seed, epoch, probe_j[i], F, 0.5)
        K = ot.unpack(grad[i], F, H)['kernel']
        for f in range(F):
            for g in range(3):
                col = K[f, g * H:(g + 1) * H]
                if keep[g, f]:
                    assert np.all(col != 0), (seed, epoch, probe_j[i], f, g)
                else:
                    assert not np.any(col), (seed, epoch, probe_j[i], f, g)
        assert 0 < np.count_nonzero(~keep) < 48
        check_grad(grad[i], want[i][1], f32[i][1], F, H, (seed, epoch, probe_j[i]))
    assert pad_ok(dw.cpu().numpy(), specs, F)


# ---- 3. optimizer, shuffle, loss bias, saturation, padding, the Python path ------------------------------------------------

def _default(fx, n=64, seed=11):
    core = fx.core('default')
    rs = np.random.RandomState(seed)
    x = rs.randn(n, core.n_features, core.feature_size).astype(np.float32)
    y = (rs.rand(n) < 0.5).astype(np.uint8)
    return core, x, y


def _f32_rmsprop(w, a, g, lr, rho, eps):
    """train_update_kernel's step in float32: a = fmaf(rho, a, (1 - rho) (g g)); w -= lr g / (sqrtf(a) + eps)."""
    f = np.float32
    c = (f(1) - f(rho)) * (g * g)
    a = (np.float64(f(rho)) * a.astype(np.float64) + c.astype(np.float64)).astype(np.float32)
    return w - f(lr) * g / (np.sqrt(a) + f(eps)), a


def _ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.abs(a - b) / np.spacing(np.maximum(np.abs(a), np.abs(b)))


@gpu
def test_shuffle_order_and_accumulator_recurrence(fx):
    """lr 0 and rho 0.5, one epoch at batch size 1: the final accumulator is the float32 recurrence over each entry's own
    gradient (pb_train_loss of that entry alone) taken in ot.shuffle's order, within 2 ulp; the weights do not move.  The
    recurrence weighs late gradients most, so another order gives another result."""
    core, x, y = _default(fx)
    F = core.feature_size
    specs = [(9, 'linear', 'hard_sigmoid', 0xDEADBEEF), (20, 'tanh', 'sigmoid', 2 ** 32 - 1)]
    n = [9, 7]
    recs = [np.asarray([3, 17, 4, 40, 41, 8, 22, 9, 63], np.int32), np.asarray([1, 2, 50, 51, 52, 5, 60], np.int32)]
    w = padded(np.random.RandomState(4).randn(2, STRIDE) * 0.2, specs, F)
    rows = core.train_rows(*[[s[c] for s in specs] for c in range(4)])
    pr = np.concatenate([np.full(c, i, np.int32) for i, c in enumerate(n)])
    pc = np.concatenate(recs)
    rms0 = np.where(w == SENTINEL, SENTINEL, np.float32(0)).astype(np.float32)
    dw, drms = fx.dev(w), fx.dev(rms0)
    loss = core.train(fx.dev(x), y, rows, dw, drms, pr, pc, epochs=1, epoch0=123456, batch_size=1, lr=0.0, rho=0.5,
                      dropout=0.0).cpu().numpy()
    assert _same(dw.cpu().numpy(), w)
    got = drms.cpu().numpy()
    assert pad_ok(got, specs, F)
    # each entry alone: one row per entry
    ones = [(s[0], s[1], s[2], s[3]) for i, s in enumerate(specs) for _ in range(n[i])]
    one_rows = core.train_rows(*[[s[c] for s in ones] for c in range(4)])
    one_w = np.concatenate([np.repeat(w[i:i + 1], n[i], 0) for i in range(2)])
    l1, g1 = core.train_loss(fx.dev(x), y, one_rows, fx.dev(one_w), np.arange(len(ones), dtype=np.int32), pc, loss_bias=0.8,
                             grad=True)
    g1, l1 = g1.cpu().numpy(), l1.cpu().numpy()
    at = 0
    for i, (H, _a, _r, s) in enumerate(specs):
        k = ot.row_size(F, H)
        order = ot.shuffle(s, 123456, n[i])
        assert sorted(order) == list(range(n[i])) and list(order) != list(range(n[i]))
        gi = g1[at:at + n[i], :k]
        acc = np.zeros(k, np.float32)
        for j in order:
            _, acc = _f32_rmsprop(np.zeros(k, np.float32), acc, gi[j], 0.0, 0.5, 1e-7)
        assert np.max(_ulps(got[i, :k], acc)) <= 2, (i, np.max(_ulps(got[i, :k], acc)))
        plain = np.zeros(k, np.float32)
        for j in range(n[i]):
            _, plain = _f32_rmsprop(np.zeros(k, np.float32), plain, gi[j], 0.0, 0.5, 1e-7)
        assert np.max(_ulps(got[i, :k], plain)) > 1000              # request order would be far off
        assert abs(loss[i, 0] - np.mean(l1[at:at + n[i]])) <= 1e-12 * abs(loss[i, 0])
        at += n[i]


@gpu
def test_one_update_follows_the_formula(fx):
    """lr 0.01, rho 0.5, eps 1e-4 and a nonzero starting accumulator, one batch: the step is RMSprop applied to the
    device's own gradient (pb_train_loss over the same entries in the shuffled order, which at dropout 0 is bit for bit
    what pb_train sums) within 2 ulp.  eps is large enough here to move the step far past 2 ulp."""
    core, x, y = _default(fx)
    F = core.feature_size
    specs = [(24, 'linear', 'hard_sigmoid', 77), (5, 'tanh', 'sigmoid', 2 ** 31), (17, 'linear', 'sigmoid', 3)]
    n = [64, 37, 130]
    rs = np.random.RandomState(8)
    recs = [rs.randint(0, len(x), c).astype(np.int32) for c in n]
    w = padded(rs.randn(3, STRIDE) * 0.2, specs, F)
    rms0 = padded(rs.uniform(1e-6, 1e-4, (3, STRIDE)), specs, F)
    rows = core.train_rows(*[[s[c] for s in specs] for c in range(4)])
    pr = np.concatenate([np.full(c, i, np.int32) for i, c in enumerate(n)])
    dw, drms = fx.dev(w), fx.dev(rms0)
    core.train(fx.dev(x), y, rows, dw, drms, pr, np.concatenate(recs), epochs=1, epoch0=9, batch_size=200, lr=0.01, rho=0.5,
               epsilon=1e-4, loss_bias=0.8, dropout=0.0)
    gw, gr = dw.cpu().numpy(), drms.cpu().numpy()
    assert pad_ok(gw, specs, F) and pad_ok(gr, specs, F)
    shuffled = np.concatenate([recs[i][ot.shuffle(s[3], 9, n[i])] for i, s in enumerate(specs)])
    _, g = core.train_loss(fx.dev(x), y, rows, dw.new_tensor(w), pr, shuffled, loss_bias=0.8, grad=True)
    g = g.cpu().numpy()
    for i, (H, *_r) in enumerate(specs):
        k = ot.row_size(F, H)
        w1, a1 = _f32_rmsprop(w[i, :k], rms0[i, :k], g[i, :k], 0.01, 0.5, 1e-4)
        assert np.max(_ulps(gr[i, :k], a1)) <= 2
        assert np.max(_ulps(gw[i, :k], w1)) <= 2, np.max(_ulps(gw[i, :k], w1))
        w7, _ = _f32_rmsprop(w[i, :k], rms0[i, :k], g[i, :k], 0.01, 0.5, 1e-7)
        assert np.max(_ulps(gw[i, :k], w7)) > 100                      # eps reaches the step


@gpu
@pytest.mark.parametrize('bias,label', [(0.0, 0), (1.0, 1)])
def test_loss_bias_ends_give_zero_gradients(fx, bias, label):
    """loss_bias 0 weighs only positives, 1 only negatives: on a batch of the other label the loss and gradient are exactly
    zero, and training leaves the weights where they were."""
    torch = fx.torch
    core, x, _ = _default(fx)
    F = core.feature_size
    y = np.full(len(x), label, np.uint8)
    specs = [(H, a, r, H) for H, (a, r) in zip((1, 13, 24, 8), ACTS)]
    w = padded(np.random.RandomState(3).randn(4, STRIDE) * 0.3, specs, F)
    rows = core.train_rows(*[[s[c] for s in specs] for c in range(4)])
    dw = fx.dev(w)
    loss, g = core.train_loss(fx.dev(x), y, rows, dw, loss_bias=bias, dropout=0.3, grad=True)
    assert not np.any(loss.cpu().numpy()) and not np.any(g.cpu().numpy())
    drms = torch.zeros_like(dw)
    loss = core.train(fx.dev(x), y, rows, dw, drms, epochs=2, batch_size=16, loss_bias=bias, dropout=0.0).cpu().numpy()
    assert not np.any(loss) and _same(dw.cpu().numpy(), w)


@gpu
@pytest.mark.parametrize('db', [40.0, -40.0])
def test_saturated_dense_layer_stays_finite(fx, db):
    """Dense bias +-40: p rounds to 1 or to 4e-18 in float32.  The loss follows float64, the gradient keeps the block rule,
    and a few epochs of training leave every weight and accumulator finite."""
    core, x, y = _default(fx)
    F = core.feature_size
    specs = [(H, a, r, 30 + H) for H, (a, r) in zip((1, 7, 24, 16), ACTS)]
    w = np.random.RandomState(6).randn(4, STRIDE) * 0.2
    for i, sp in enumerate(specs):
        w[i, ot.row_size(F, sp[0]) - 1] = db
    w = padded(w, specs, F)
    rows = core.train_rows(*[[s[c] for s in specs] for c in range(4)])
    dw = fx.dev(w)
    loss, g = core.train_loss(fx.dev(x), y, rows, dw, loss_bias=0.8, grad=True)
    loss, g = loss.cpu().numpy(), g.cpu().numpy()
    masks = Masks()
    allr = [np.arange(len(x))] * 4
    want = oracle(specs, w, x, y, allr, F, 0.0, 0, 0.8, masks, np.float64)
    f32 = oracle(specs, w, x, y, allr, F, 0.0, 0, 0.8, masks, np.float32)
    jump = jumps(specs, w, x, y, allr, F, 0.0, 0, 0.8, masks)
    for i, (H, *_r) in enumerate(specs):
        check_loss(loss[i], want[i][0], f32[i][0], (db, H))
        check_grad(g[i], want[i][1], f32[i][1], F, H, (db, H), jump[i])
    drms = fx.dev(padded(np.zeros((4, STRIDE)), specs, F))
    tl = core.train(fx.dev(x), y, rows, dw, drms, epochs=3, batch_size=16).cpu().numpy()
    assert np.all(np.isfinite(tl)) and np.all(np.isfinite(dw.cpu().numpy())) and np.all(np.isfinite(drms.cpu().numpy()))
    assert pad_ok(dw.cpu().numpy(), specs, F) and pad_ok(drms.cpu().numpy(), specs, F)


@gpu
def test_offline_train_is_the_direct_calls(fx):
    """offline.train with sensitivity, lr, dropout and a pair validation set is, bit for bit, core.train one epoch at a time
    (loss_bias = 1 - sensitivity, epoch0 advancing) followed by core.train_loss at dropout 0."""
    torch = fx.torch
    m = fx.m
    core, x, y = _default(fx, n=96)
    F = core.feature_size
    specs = [(20, 'linear', 'hard_sigmoid', 5), (3, 'tanh', 'sigmoid', 2 ** 32 - 1), (11, 'tanh', 'hard_sigmoid', 9)]
    w = padded(np.random.RandomState(12).randn(3, STRIDE) * 0.2, specs, F)
    rs = np.random.RandomState(13)
    pr = rs.randint(0, 3, 150).astype(np.int32)
    pc = rs.randint(0, 64, 150).astype(np.int32)
    vr = rs.randint(0, 3, 40).astype(np.int32)
    vc = rs.randint(64, 96, 40).astype(np.int32)
    dx = fx.dev(x)
    kw = dict(sensitivity=0.3, lr=0.01, dropout=0.25, batch_size=32)
    st = m.offline.TrainState(core, fx.dev(w), fx.dev(padded(np.zeros((3, STRIDE)), specs, F)), [s[0] for s in specs],
                              [s[1] for s in specs], [s[2] for s in specs], [s[3] for s in specs], epoch=4)
    loss, val = m.offline.train(core, st, dx, y, pr, pc, epochs=3, validation=(dx, y, vr, vc), **kw)
    assert st.epoch == 7
    rows = core.train_rows(*[[s[c] for s in specs] for c in range(4)])
    dw, drms = fx.dev(w), fx.dev(padded(np.zeros((3, STRIDE)), specs, F))
    ls, vs = [], []
    for e in range(4, 7):
        ls.append(core.train(dx, y, rows, dw, drms, pr, pc, epochs=1, epoch0=e, batch_size=32, lr=0.01, rho=0.9, epsilon=1e-7,
                             loss_bias=1.0 - 0.3, dropout=0.25))
        vs.append(core.train_loss(dx, y, rows, dw, vr, vc, loss_bias=1.0 - 0.3, dropout=0.0))
    assert _same(loss, torch.cat(ls, 1).cpu().numpy()) and _same(val, torch.stack(vs, 1).cpu().numpy())
    assert _same(st.weights.cpu().numpy(), dw.cpu().numpy()) and _same(st.rms.cpu().numpy(), drms.cpu().numpy())
    assert pad_ok(dw.cpu().numpy(), specs, F) and pad_ok(drms.cpu().numpy(), specs, F)
    assert not _same(dw.cpu().numpy(), w)


# ---- 4. hard_sigmoid's bounds ----------------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize('front', ['t1', 'default'])
def test_hard_sigmoid_gradient_at_its_bounds(fx, front):
    """The z gate's pre-activation is its bias at every step: at T = 1 all-zero inputs and a zero recurrent kernel; at
    T = 29 random inputs with zero z-gate kernel columns, zero z and r recurrent blocks and a random candidate block, which
    carries dh back through the steps.  At -2.5 Keras's 0.2 x + 0.5 is exactly 0, the lower bound, where the gradient is 0.2
    in float64 and float32: the z-gate gradient dh (h_prev - candidate) 0.2 must be that, not 0.  At 2.5, the upper
    bound, likewise."""
    core = fx.core(front)
    F, T = core.feature_size, core.n_features
    x = np.zeros((3, T, F), np.float32) if T == 1 else np.random.RandomState(0).randn(3, T, F).astype(np.float32)
    y = np.ones(3, np.uint8)
    specs, w = [], []
    for bz in (-2.5, 2.5):
        for H, act in ((1, 'linear'), (5, 'tanh'), (24, 'linear')):
            rs = np.random.RandomState(H)
            row = np.zeros(STRIDE, np.float32)
            p = ot.unpack(row, F, H)
            p['kernel'][:, H:] = rs.randn(F, 2 * H) * 0.3
            if T > 1:
                p['recurrent'][:, 2 * H:] = rs.randn(H, H) * 0.3
            p['bias'][:H] = bz
            p['bias'][H:2 * H] = rs.randn(H) * 0.5
            p['bias'][2 * H:] = 0.7
            p['dense_w'][...] = rs.uniform(0.5, 1.0, H) * rs.choice([-1, 1], H)
            row[ot.row_size(F, H) - 1] = 0.1
            specs.append((H, act, 'hard_sigmoid', 1))
            w.append(row)
    w = padded(np.stack(w), specs, F)
    rows = core.train_rows(*[[s[c] for s in specs] for c in range(4)])
    _, g = core.train_loss(fx.dev(x), y, rows, fx.dev(w), loss_bias=0.8, grad=True)
    g = g.cpu().numpy()
    masks = Masks()
    allr = [np.arange(3)] * len(specs)
    want = oracle(specs, w, x, y, allr, F, 0.0, 0, 0.8, masks, np.float64)
    f32 = oracle(specs, w, x, y, allr, F, 0.0, 0, 0.8, masks, np.float32)
    for i, (H, *_r) in enumerate(specs):
        bz = float(w[i, ot.row_size(F, H) - 1 - H - 3 * H])
        dz, d64, d32 = (_blocks(v, F, H)['bias z'] for v in (g[i], want[i][1], f32[i][1]))
        assert np.all(d64 != 0) and np.all(d32 != 0), (front, bz, H)
        assert np.all(dz != 0), (front, bz, H, dz, d64)
        bound = 10 * np.max(np.abs(d32 - d64)) + 1e-6 * np.max(np.abs(d64))
        assert np.max(np.abs(dz - d32)) <= bound, (front, bz, H, dz, d32)
        check_grad(g[i], want[i][1], f32[i][1], F, H, (front, bz, H))


# ---- 5. several workspace groups -------------------------------------------------------------------------------------------

def group_cost(n, bs):
    """train_groups' bytes for a row of n entries at batch size bs (csrc/api.cu): 40 per entry, one partial gradient row
    (2 980 floats + a double) per tile of the largest batch, 20 per tile and per batch, 64 of slack."""
    b, nb = min(bs, n), -(-n // bs)
    tiles = sum(-(-min(bs, n - b0) // TILE) for b0 in range(0, n, bs))
    return n * 40 + -(-b // TILE) * (STRIDE * 4 + 8) + tiles * 20 + nb * 20 + 64


def n_groups(ns, bs):
    out, acc = 0, 0
    for n in ns:
        if n == 0:
            continue
        c = group_cost(n, bs)
        if out == 0 or acc + c > WS_CAP:
            out, acc = out + 1, 0
        acc += c
    return out


def _many(fx, core, specs, w):
    rows = core.train_rows(*[[s[c] for s in specs] for c in range(4)])
    return rows, fx.dev(w), fx.dev(padded(np.zeros_like(w), specs, core.feature_size))


@gpu
def test_pairs_over_three_groups_equal_single_group_chunks(fx):
    """About 50 000 one-entry rows by pairs: a one-entry row costs 12 072 bytes of arena, so 22 236 rows fill a 256 MB
    group and the call runs as three groups.  Rows without entries sit at both group boundaries and at the ends.  Weights,
    accumulators, losses (pb_train) and losses and gradients (pb_train_loss) are bit-identical to the same rows in calls of
    at most 20 000 rows, each a single group."""
    core = fx.core('default')
    F, T = core.feature_size, core.n_features
    assert group_cost(1, 16) == 12072 and WS_CAP // 12072 == 22236
    n_full = 50000
    # row index -> entries: one each, except empty rows around the boundaries after 22 236 and 44 472 rows with entries
    ns = [0]
    for i in range(n_full):
        if i in (22236, 44472):
            ns += [0, 0]
        ns.append(1)
    ns.append(0)
    assert n_groups(ns, 16) == 3 and n_groups(ns, 1 << 40) == 3
    k = len(ns)
    specs = [(HIDDEN[i % len(HIDDEN)], *ACTS[(i // 3) % 4], i) for i in range(k)]
    rs = np.random.RandomState(21)
    w = np.random.default_rng(rs.randint(1 << 30)).standard_normal((k, STRIDE), dtype=np.float32) * np.float32(0.2)
    size = np.asarray([ot.row_size(F, s[0]) for s in specs])
    w[np.arange(STRIDE)[None, :] >= size[:, None]] = SENTINEL
    x = rs.randn(512, T, F).astype(np.float32)
    y = (rs.rand(512) < 0.5).astype(np.uint8)
    dx = fx.dev(x)
    pr = np.asarray([i for i, c in enumerate(ns) if c], np.int32)
    pc = (pr * 7 % 512).astype(np.int32)
    empty = [i for i, c in enumerate(ns) if c == 0]
    assert len(empty) == 6 and empty[0] == 0 and empty[-1] == k - 1
    rows, dw, drms = _many(fx, core, specs, w)
    loss = core.train(dx, y, rows, dw, drms, pr, pc, epochs=2, epoch0=3, batch_size=16, lr=0.003, dropout=0.2)
    l_loss, l_grad = core.train_loss(dx, y, rows, fx.dev(w), pr, pc, loss_bias=0.6, dropout=0.1, epoch=4, grad=True)
    got = [dw.cpu().numpy(), drms.cpu().numpy(), loss.cpu().numpy(), l_loss.cpu().numpy(), l_grad.cpu().numpy()]
    del dw, drms, l_grad
    assert np.all(np.isnan(got[2][empty])) and np.all(np.isnan(got[3][empty]))
    assert _same(got[0][empty], w[empty]) and np.all(got[1][empty][w[empty] != SENTINEL] == 0)
    assert np.all(np.isfinite(got[2][pr])) and np.all(np.isfinite(got[4]))
    assert np.all(got[0][w == SENTINEL] == SENTINEL) and np.all(got[1][w == SENTINEL] == SENTINEL)
    for c0 in range(0, k, 20000):
        c1 = min(k, c0 + 20000)
        sel = (pr >= c0) & (pr < c1)
        assert n_groups(ns[c0:c1], 16) == 1
        rows, dw, drms = _many(fx, core, specs[c0:c1], w[c0:c1])
        loss = core.train(dx, y, rows, dw, drms, pr[sel] - c0, pc[sel], epochs=2, epoch0=3, batch_size=16, lr=0.003, dropout=0.2)
        assert _same(dw.cpu().numpy(), got[0][c0:c1]) and _same(drms.cpu().numpy(), got[1][c0:c1])
        assert _same(loss.cpu().numpy(), got[2][c0:c1])
        l_loss, l_grad = core.train_loss(dx, y, rows, fx.dev(w[c0:c1]), pr[sel] - c0, pc[sel], loss_bias=0.6, dropout=0.1,
                                         epoch=4, grad=True)
        assert _same(l_loss.cpu().numpy(), got[3][c0:c1]) and _same(l_grad.cpu().numpy(), got[4][c0:c1])


@gpu
def test_cross_product_over_two_groups_equals_single_group_chunks(fx):
    """300 rows x 5 000 clips at batch size 5 000: about 1.14 MB of arena per row (40 bytes per entry and 79 tiles'
    partials), 234 rows per group, two groups.  Bit-identical to two calls of 150 rows."""
    core = fx.core('default')
    F, T = core.feature_size, core.n_features
    n, k = 5000, 300
    assert group_cost(n, n) == 1143976 and WS_CAP // 1143976 == 234 and n_groups([n] * k, n) == 2
    rs = np.random.RandomState(31)
    x = rs.randn(n, T, F).astype(np.float32)
    y = (rs.rand(n) < 0.3).astype(np.uint8)
    dx = fx.dev(x)
    specs = [(HIDDEN[i % len(HIDDEN)], *ACTS[i % 4], 1000 + i) for i in range(k)]
    w = np.random.default_rng(rs.randint(1 << 30)).standard_normal((k, STRIDE), dtype=np.float32) * np.float32(0.2)
    w = padded(w, specs, F)
    rows, dw, drms = _many(fx, core, specs, w)
    loss = core.train(dx, y, rows, dw, drms, epochs=1, epoch0=1, batch_size=n, lr=0.002, dropout=0.2)
    l_loss, l_grad = core.train_loss(dx, y, rows, fx.dev(w), loss_bias=0.7, dropout=0.2, epoch=2, grad=True)
    got = [dw.cpu().numpy(), drms.cpu().numpy(), loss.cpu().numpy(), l_loss.cpu().numpy(), l_grad.cpu().numpy()]
    assert not _same(got[0], w) and pad_ok(got[0], specs, F) and pad_ok(got[1], specs, F)
    for c0 in (0, 150):
        rows, dw, drms = _many(fx, core, specs[c0:c0 + 150], w[c0:c0 + 150])
        loss = core.train(dx, y, rows, dw, drms, epochs=1, epoch0=1, batch_size=n, lr=0.002, dropout=0.2)
        assert _same(dw.cpu().numpy(), got[0][c0:c0 + 150]) and _same(drms.cpu().numpy(), got[1][c0:c0 + 150])
        assert _same(loss.cpu().numpy(), got[2][c0:c0 + 150])
        l_loss, l_grad = core.train_loss(dx, y, rows, fx.dev(w[c0:c0 + 150]), loss_bias=0.7, dropout=0.2, epoch=2, grad=True)
        assert _same(l_loss.cpu().numpy(), got[3][c0:c0 + 150]) and _same(l_grad.cpu().numpy(), got[4][c0:c0 + 150])


# ---- 6. refusals and the row-size limit -----------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize('kw', [dict(buffer_t=5.7), dict(hop_t=0.005)], ids=['t113', 't281'])
def test_front_ends_past_the_kernel_are_refused(fx, kw):
    """T = 113 needs 233 168 bytes of shared memory, past the 232 448 a CTA may have; T = 281 far more.  All three calls
    raise NotImplementedError (PB_ERR_UNSUPPORTED), and the weights and accumulators stay as they were."""
    torch = fx.torch
    m = fx.m
    core = m.PreciseB200(m.ListenerParams(**kw))
    try:
        F, T = core.feature_size, core.n_features
        assert T in (113, 281)
        specs = [(20, 'linear', 'hard_sigmoid', 1)]
        w = padded(np.random.RandomState(1).randn(1, STRIDE) * 0.2, specs, F)
        rows, dw, drms = _many(fx, core, specs, w)
        drms.fill_(0.25)
        r0 = drms.cpu().numpy()
        dx = torch.zeros((2, T, F), dtype=torch.float32, device='cuda')
        with pytest.raises(NotImplementedError):
            core.vectorize_clips(fx.dev(np.ones(4000, np.int16)), np.asarray([0, 4000], np.int64))
        with pytest.raises(NotImplementedError):
            core.train(dx, np.ones(2, np.uint8), rows, dw, drms, epochs=1)
        with pytest.raises(NotImplementedError):
            core.train_loss(dx, np.ones(2, np.uint8), rows, dw, grad=True)
        torch.cuda.synchronize()
        assert _same(dw.cpu().numpy(), w) and _same(drms.cpu().numpy(), r0)
    finally:
        core.close()


@gpu
def test_row_size_limit(fx):
    """A row may have at most 2^22 = 4 194 304 entries (256 MB / 64).  One more is refused by both calls and changes
    nothing.  At the limit the call runs (its arena, about 950 MB, is past 256 MB: one row's partials are not split), and
    since every entry is the same clip the row's loss is that clip's loss exactly."""
    torch = fx.torch
    core, x, y = _default(fx, n=4)
    F = core.feature_size
    specs = [(1, 'linear', 'hard_sigmoid', 1), (4, 'tanh', 'sigmoid', 2)]
    w = padded(np.random.RandomState(2).randn(2, STRIDE) * 0.2, specs, F)
    rows, dw, drms = _many(fx, core, specs, w)
    drms.fill_(0.5)
    r0 = drms.cpu().numpy()
    dx = fx.dev(x)
    lim = 1 << 22
    pr = np.zeros(lim + 1, np.int32)
    pc = np.full(lim + 1, 2, np.int32)
    pr[-1] = 1
    pc[-1] = 3
    over = np.zeros(lim + 1, np.int32)
    with pytest.raises(ValueError):
        core.train(dx, y, rows, dw, drms, over, pc, epochs=1)
    with pytest.raises(ValueError):
        core.train_loss(dx, y, rows, dw, over, pc, grad=True)
    torch.cuda.synchronize()
    assert _same(dw.cpu().numpy(), w) and _same(drms.cpu().numpy(), r0)
    big = core.train_loss(dx, y, rows, dw, pr, pc).cpu().numpy()
    one = core.train_loss(dx, y, rows, dw, np.asarray([0, 1], np.int32), np.asarray([2, 3], np.int32)).cpu().numpy()
    assert big[0] == one[0] and big[1] == one[1], (big, one)
