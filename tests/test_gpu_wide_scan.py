"""The wide networks' GRU scans against the float64 GRU, over the shapes, front ends, weight magnitudes and call paths that
reach them; and the default network's CUDA-core scans under the same rules.

Every network that is not the default one (H 20, F 13, Keras's activations) and not of the fused family on a bank or pool
path runs one of two kernels (launch_gru_kernels in api.cu): gru_wide_kernel (gru_wide.cuh, mma.sync 3 x TF32) for H <= 128
and feature size F <= 40, gru_tiled_kernel (gru_kernels.cuh, CUDA-core SGEMM) for everything up to F + 3H = 800 and for
every network under gru_mode 1.  The default network runs gru_warp_kernel<20, 13> (up to 8 192 items) or, under gru_mode 1,
gru_small_kernel<20, 13> (its ROUTE instantiation on routed ticks).  Each output here is anchored to oracle.gru.gru_forward
in float64 (p64) on the window the GPU itself scored: pb_predict's own input, or read_window after a tick with
oracle.mfcc.add_deltas applied for delta front ends, which isolates the scan from the MFCC front end.

- Shapes: feature sizes 13 to 128 (MFCCs, 64 log-mels and speechpy MFCCs, with and without deltas; 41 and 128 only on the
  tiled kernel, whose ring rows are then 44 and 64 floats apart), window lengths T = 1, 29, 73 and 281, hidden sizes 1 ..
  128 on both kernels (HP / 16 = 1 .. 8 active warps of gru_wide_kernel, partial last warps), 129 .. 262 on the tiled kernel
  (a second phase-1 column chunk from H 129, a second phase-2 chunk from H 257), and on every front end the largest H with
  F + 3H <= 800, which is 800 exactly where 800 - F is a multiple of 3.  All four activation pairs rotate over the grid.
- Weight families: std 0.1 / sqrt(H / 20), Keras-initialiser-like weights (glorot-uniform kernel, orthogonal recurrent
  blocks, zero bias) at gain 1 and 1.3, tanh / sigmoid networks at gain 2 and 3, and doubling networks (h_t = 2 h + 1, h near
  2^T, inside float32's range for T <= 100) whose raw must be float64's saturated decision, 1.0 or 0.0, exactly.  No trained
  Precise model ships with the reference and none can be fetched, so "trained-like" is an assumption built from Keras's
  default initialisers.
- Bounds: per output, where the float32 GRU (p32) is within 1e-6 of float64, |raw - p64| < 1e-5.  Over the outputs of one
  call (a case's windows), max |raw - p64| <= 4 max |p32 - p64| + 1e-6 on the CUDA-core kernels, 2 max |p_f16x3 - p64| +
  2 max |p32 - p64| + 1e-6 on fused bank slots, and 4 max |p_tf32x3 - p64| + 4 max |p32 - p64| + 2e-6 on gru_wide_kernel
  (p_tf32x3 = oracle.gru.gru_forward_tf32x3).  pb_predict's logit obeys the same rules relative to max(1, |l64|), with
  test_gpu_fused_scan.py's logit constants (4e-6 / 5e-5; 8e-6 on gru_wide_kernel).  Measured exceptions to the rule
  the fused scan meets (DESIGN.md section 6, "Wide and tiled accuracy"): the relative rule is applied to a call's worst
  output rather than to each output, because one output's float32 error is a single sample and can be small by chance
  (per output, the first H100 run failed it by up to 1.2e-5 on the tiled kernel and 1.3e-6 on the wide one); CHAOTIC; and
  gru_wide_kernel gets factors 4 and twice the constant, because its tensor cores round each m16n8k8 accumulation in
  float32 (3 per k-step, up to 63 per gate and step), which p_tf32x3, summing exactly, does not model.  check() records each
  wide call's ratio to the fused rule and report() prints the worst; on the H100 the cases past 1 were one-model ticks on
  the default front end, Keras gain 1.3, H 64 (raw, 1.21) and pb_predict on 20 MFCCs + deltas, Keras gain 1.3, H 24
  (logit, 1.47).
- Call paths: pb_predict at N = 1 .. 300 and 10 000 (checked on a strided sample), both kernel modes for every network
  gru_wide_kernel accepts; one-model ticks, routed and not, in both modes; a bank mixing fused and non-fused slots, routed
  and not, with per-stream trigger settings on one slot; ragged ticks; pb_score_corpus against the stream ticks and the
  oracle listener; and the refusals at F + 3H = 801.

-m gpu throughout."""
import numpy as np
import pytest

from oracle import gru as og
from oracle.listener import run_streams
from oracle.mfcc import add_deltas
from oracle.params import OracleParams
from oracle.trigger import OracleTrigger

gpu = pytest.mark.gpu
CHUNK = 2048
TICKS = 14                 # 28 672 samples: every window here fills, and the first ticks score young windows
CHECKED = (0, 1, 4, 8, 13)  # ticks compared with float64 (every tick is scored and its trigger replayed)
ACTS = (('linear', 'hard_sigmoid'), ('tanh', 'sigmoid'), ('linear', 'sigmoid'), ('tanh', 'hard_sigmoid'))
WIDE_H = (1, 7, 17, 24, 25, 31, 32, 33, 48, 63, 64, 65, 81, 96, 100, 112, 113, 127, 128)   # HP / 16 = 1 .. 8
TILED_H = (129, 160, 200, 255, 256, 257, 262)
BATCHES = (1, 63, 64, 65, 127, 128, 129, 300)
BIG = 10000
# Measured exception: over T = 281 steps the tanh / sigmoid networks at gain 3 diverge from float64 in float32 itself.  On
# the H100, with the bounds below, pb_predict's tiled logit there was 1.4e-3 (relative) past its bound and a one-model tick's
# wide raw 1.2e-5 past its (factor-4) bound.  That family runs at T <= CHAOTIC[1] only; every other family runs at T = 281.
CHAOTIC = ('tanh/sigmoid 3', 100)
ROUTE_AT = 5                # routed handles clear bit 0 on some streams before this tick: their triggers hold state by then


def _mod():
    import mycroft_precise_b200 as m
    return m


def cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


FRONT_ENDS = {                 # name: ListenerParams arguments (F = feature size, T = n_features)
    'default': {},                                                      # F 13, T 29
    'delta': dict(use_delta=True),                                      # F 26
    'f17': dict(n_filt=20, n_mfcc=17),                                  # F 17
    'config3': dict(n_filt=40, n_mfcc=40),                              # F 40: gru_wide_kernel's limit
    'delta20': dict(n_mfcc=20, use_delta=True),                         # F 40
    'f41': dict(n_filt=41, n_mfcc=41),                                  # F 41: tiled only
    'mels64d': dict(vectorizer=1, n_filt=64, n_mfcc=64, use_delta=True),  # F 128, ring rows 64 floats apart: tiled only
    'speechpy_d': dict(vectorizer=3, use_delta=True),                   # F 26
    'd_t1': dict(use_delta=True, buffer_t=0.1),                         # T 1
    'd_t73': dict(use_delta=True, hop_t=0.02, window_t=0.05),           # T 73
    'd_t281': dict(use_delta=True, hop_t=0.005),                        # T 281
}


def params(name):
    return _mod().ListenerParams(**FRONT_ENDS[name])


def limit_h(F):
    """The largest H gru_tiled_kernel accepts at feature size F (F + 3H <= 800)."""
    return (800 - F) // 3


def wide_ok(F, H):
    return H <= 128 and F <= 40


def audio(S, n, seed):
    """Stream s: noise at sigma 30 / 300 / 3000 / 12 000, silence, +32767, -32768 or a full-scale square wave (s % 8)."""
    rs = np.random.RandomState(seed)
    pcm = np.zeros((S, n), np.int16)
    for s in range(S):
        kind = s % 8
        if kind < 4:
            pcm[s] = np.clip(rs.randn(n) * (30, 300, 3000, 12000)[kind], -32768, 32767)
        elif kind == 5:
            pcm[s] = 32767
        elif kind == 6:
            pcm[s] = -32768
        elif kind == 7:
            pcm[s] = np.where((np.arange(n) // 37) % 2, 32767, -32767)
    return pcm


def weights(model):
    return og.GruWeights(model.kernel, model.recurrent, model.bias, model.dense_w, model.dense_b,
                         model.activation, model.recurrent_activation)


def keras_like(F, H, seed, gain, act=ACTS[0]):
    """Keras's default GRU initialisers times ``gain``: glorot-uniform kernel and dense weights, an orthogonal block per gate
    of the recurrent kernel, zero biases."""
    m = _mod()
    rs = np.random.RandomState(seed)
    lim = np.sqrt(6.0 / (F + 3 * H))
    kernel = rs.uniform(-lim, lim, (F, 3 * H))
    rec = np.concatenate([np.linalg.qr(rs.randn(H, H))[0] for _ in range(3)], axis=1)
    lim = np.sqrt(6.0 / (H + 1))
    g = m.GruModel(gain * kernel, gain * rec, np.zeros(3 * H), gain * rs.uniform(-lim, lim, H), 0.0)
    g.activation, g.recurrent_activation = act
    return g


def doubling(F, H, sign, act=ACTS[0]):
    """z = 0, r = 1, candidate recurrent block 2 I, candidate bias 1: h_t = 2 h_(t-1) + 1 in every unit, whatever the input.
    The Dense layer, sign (1e-4 sum(h) / H - 2), is past float32 sigmoid's saturation once h is past 10^6 (T >= 20)."""
    m = _mod()
    rec = np.zeros((H, 3 * H))
    rec[:, 2 * H:] = 2 * np.eye(H)
    bias = np.concatenate([np.full(H, -10.0), np.full(H, 10.0), np.ones(H)])
    g = m.GruModel(np.zeros((F, 3 * H)), rec, bias, np.full(H, 1e-4 * sign / H), -2.0 * sign)
    g.activation, g.recurrent_activation = act
    return g


def std_model(F, H, seed, act):
    g = _mod().GruModel.random(F, H, seed=seed, scale=0.1 / np.sqrt(max(H, 20) / 20.0))   # contractive recurrence
    g.activation, g.recurrent_activation = act
    return g


FAMILIES = {
    'std': lambda F, H, seed, act: std_model(F, H, seed, act),
    'keras 1': lambda F, H, seed, act: keras_like(F, H, seed, 1.0, act),
    'keras 1.3': lambda F, H, seed, act: keras_like(F, H, seed, 1.3, act),
    'tanh/sigmoid 2': lambda F, H, seed, act: keras_like(F, H, seed, 2.0, ACTS[1]),
    'tanh/sigmoid 3': lambda F, H, seed, act: keras_like(F, H, seed, 3.0, ACTS[1]),
    'doubling +': lambda F, H, seed, act: doubling(F, H, 1.0, act if act[0] == 'linear' else ACTS[0]),
    'doubling -': lambda F, H, seed, act: doubling(F, H, -1.0, act if act[0] == 'linear' else ACTS[0]),
}


def saturates(g, T):
    """A doubling network whose float64 decision is saturated at window length T."""
    return g.dense_b != 0 and np.all(g.kernel == 0) and T >= 20


# ------------------------------------------------------------------------------------------------------------ references
def refs(w, x, kind):
    """(p, logit) of float64, float32 and the kernel's own reference (tf32x3 for 'wide', f16x3 for 'fused', None else)."""
    with np.errstate(over='ignore'):
        r = {'64': og.gru_forward(w, x, np.float64), '32': og.gru_forward(w, x, np.float32)}
        r['k'] = og.gru_forward_tf32x3(w, x) if kind == 'wide' else og.gru_forward_f16x3(w, x) if kind == 'fused' else None
    return r


def check(raw, logit, r, kind, g, T, tag, stats, sel=slice(None)):
    """The module docstring's bounds on raw (and logit unless None) of one call against references r; records the worst
    (|raw - p64|, |p_k - p64|, |p32 - p64|) under ``tag``."""
    raw = np.asarray(raw, np.float64)
    p64, p32 = r['64'][0][sel].astype(np.float64), r['32'][0][sel].astype(np.float64)
    assert np.all(np.isfinite(raw)), (tag, 'non-finite raw')
    e, e32 = np.abs(raw - p64), np.abs(p32 - p64)
    ek = np.abs(r['k'][0][sel].astype(np.float64) - p64) if r['k'] is not None else np.zeros_like(e)
    if saturates(g, T):
        want = 1.0 if g.dense_b < 0 else 0.0
        assert np.all(np.abs(p64 - want) < 1e-12) and np.all(raw == want), (tag, np.unique(raw))
        if logit is not None:
            assert np.all(np.sign(logit) == (1 if want else -1)), tag
    else:
        tight = e32 < 1e-6
        assert np.all(e[tight] < 1e-5), (tag, float(e[tight].max()))
        lim = 4 * ek.max() + 4 * e32.max() + 2e-6 if kind == 'wide' else 2 * ek.max() + 2 * e32.max() + 1e-6 \
            if kind == 'fused' else 4 * e32.max() + 1e-6
        assert e.max() <= lim, (tag, float(e.max() - lim), float(e.max()))
        if kind == 'wide':          # what the factor-4 exception buys: the worst ratio to the fused scan's rule
            stats['_fused rule'] = max(stats.get('_fused rule', (0.0, '')),
                                       (e.max() / (2 * ek.max() + 2 * e32.max() + 1e-6), '%s H %d' % (tag, g.hidden)))
        if logit is not None:
            lg = np.asarray(logit, np.float64)
            l64 = r['64'][1][sel].astype(np.float64)
            el, el32 = np.abs(lg - l64), np.abs(r['32'][1][sel].astype(np.float64) - l64)
            elk = np.abs(r['k'][1][sel].astype(np.float64) - l64) if r['k'] is not None else np.zeros_like(el)
            assert np.all(np.isfinite(lg)), tag
            scale = np.maximum(1.0, np.abs(l64))
            tight = el32 < 4e-6 * scale
            assert np.all(el[tight] < 5e-5 * scale[tight]), (tag, 'logit', float(np.max(el[tight] / scale[tight])))
            rel, rel32 = el / scale, el32 / scale
            lim = 4 * (elk / scale).max() + 4 * rel32.max() + 8e-6 if kind == 'wide' else \
                (2 * (elk / scale).max() + 2 * rel32.max() if kind == 'fused' else 4 * rel32.max()) + 4e-6
            assert rel.max() <= lim, (tag, 'logit', float(rel.max() - lim))
            if kind == 'wide':
                stats['_fused rule, logit'] = max(stats.get('_fused rule, logit', (0.0, '')), (
                    rel.max() / (2 * (elk / scale).max() + 2 * rel32.max() + 4e-6), '%s H %d' % (tag, g.hidden)))
    if e.size:
        s = stats.setdefault(tag, np.zeros(3))
        stats[tag] = np.maximum(s, [e.max(), ek.max(), e32.max()])


def report(title, stats):
    for tag, v in sorted(stats.items()):
        if tag.startswith('_'):
            print('%s: gru_wide_kernel against the %s (2 |p_tf32x3 - p64| + 2 |p32 - p64| + 1e-6): worst ratio %.2f, %s'
                  % (title, tag[1:], v[0], v[1]))
        else:
            print('%s %s: |raw - p64| %.2g, |p_kernel - p64| %.2g, |p32 - p64| %.2g' % ((title, tag) + tuple(v)))


def kernel_of(F, H, mode, small=False):
    if small:
        return 'warp' if mode == 0 else 'small'
    return 'wide' if wide_ok(F, H) and mode == 0 else 'tiled'


def modes(F, H):
    return (0, 1) if wide_ok(F, H) else (0,)


def predictor(pr, g):
    m = _mod()
    core = m.PreciseB200(pr, hidden=g.hidden, activation=g.activation, recurrent_activation=g.recurrent_activation)
    core.load_weights(g.kernel, g.recurrent, g.bias, g.dense_w, g.dense_b)
    return core


def read_windows(core, pr, n):
    """[n, T, F] windows of streams 0..n-1 as the scan read them: MFCC rows, with deltas for delta front ends."""
    Fb = pr.feature_size // 2 if pr.use_delta else pr.feature_size
    win = core.read_window(n).cpu().numpy()[..., :Fb].astype(np.float32)
    return np.stack([add_deltas(w) for w in win]) if pr.use_delta else win


_WINDOWS = {}


def front_windows(front):
    """Every window 64 streams of ``audio`` score over TICKS ticks of this front end (young windows included)."""
    if front not in _WINDOWS:
        m = _mod()
        pr = params(front)
        S = 64
        sb = m.StreamBatch(std_model(pr.feature_size, 32, 1, ACTS[0]), S, params=pr, chunk_samples=CHUNK)
        pcm = audio(S, TICKS * CHUNK, seed=3)
        out = []
        for k in range(TICKS):
            sb.update(cuda(pcm[:, k * CHUNK:(k + 1) * CHUNK]))
            out.append(read_windows(sb.core, pr, S))
        sb.core.close()
        _WINDOWS[front] = np.concatenate(out)
    return _WINDOWS[front]


# ------------------------------------------------------------------------------------------------------------ pb_predict
def predict_case(pr, g, x, stats, tag_prefix, sample=None):
    F, T = pr.feature_size, pr.n_features
    core = predictor(pr, g)
    xs = x if sample is None else x[sample]
    kinds = {kernel_of(F, g.hidden, mode) for mode in modes(F, g.hidden)}
    r = refs(weights(g), xs, 'wide' if 'wide' in kinds else None)
    rt = dict(r, k=None)
    for mode in modes(F, g.hidden):
        core.gru_mode(mode)
        p, lg = core.predict(cuda(x), want_logit=True)
        p, lg = p.cpu().numpy(), lg.cpu().numpy()
        if sample is not None:
            p, lg = p[sample], lg[sample]
        kind = kernel_of(F, g.hidden, mode)
        check(p, lg, r if kind == 'wide' else rt, kind, g, T, '%s %s H %d N %d' % (tag_prefix, kind, g.hidden, len(x)), stats)
    core.close()


@gpu
@pytest.mark.parametrize('front', list(FRONT_ENDS))
def test_predict_shape_grid(front):
    """std networks of every hidden size (WIDE_H, TILED_H on the default front end, the front end's largest), activation pairs
    and batch sizes rotating, in both kernel modes; one batch of 10 000 windows checked every 41st."""
    pr = params(front)
    F = pr.feature_size
    fi = list(FRONT_ENDS).index(front)
    x_all = front_windows(front)
    rs = np.random.RandomState(fi)
    hs = list(WIDE_H) + (list(TILED_H) if front == 'default' else []) + [limit_h(F)]
    stats = {}
    for i, H in enumerate(hs):
        g = std_model(F, H, 100 + i, ACTS[(i + fi) % 4])
        N = BATCHES[(i + fi) % len(BATCHES)]
        predict_case(pr, g, x_all[rs.choice(len(x_all), N, replace=False)], stats, front)
    big = x_all[rs.randint(0, len(x_all), BIG)]
    predict_case(pr, std_model(F, 65, 7, ACTS[fi % 4]), big, stats, front, sample=np.arange(0, BIG, 41))
    worst = {}
    for tag, v in stats.items():
        if tag.startswith('_'):
            continue
        k = tag.split()[1]
        worst[k] = np.maximum(worst.get(k, 0), v)
    report(front, dict(worst, **{k: v for k, v in stats.items() if k.startswith('_')}))
    assert len(stats) >= len(hs) + 1


@gpu
@pytest.mark.parametrize('front', list(FRONT_ENDS))
def test_predict_weight_families(front):
    """Every weight family at a spread of hidden sizes (1 .. 8 active warps, the tiled kernel's largest), 200 windows each,
    in both kernel modes.  Prints the worst errors per kernel and family (DESIGN.md section 6)."""
    pr = params(front)
    F = pr.feature_size
    x_all = front_windows(front)
    x = x_all[np.random.RandomState(5).choice(len(x_all), 200, replace=False)]
    hs = (24, 64, 128, limit_h(F)) + ((200,) if front == 'default' else ())
    stats = {}
    for fam, make in FAMILIES.items():
        if fam.startswith('doubling') and pr.n_features > 100:      # h near 2^T leaves float32's range
            continue
        if fam == CHAOTIC[0] and pr.n_features > CHAOTIC[1]:
            continue
        for i, H in enumerate(hs):
            g = make(F, H, 300 + i, ACTS[i % 4])
            core = predictor(pr, g)
            kinds = [kernel_of(F, H, mode) for mode in modes(F, H)]
            r = refs(weights(g), x, 'wide' if 'wide' in kinds else None)
            for mode, kind in zip(modes(F, H), kinds):
                core.gru_mode(mode)
                p, lg = core.predict(cuda(x), want_logit=True)
                check(p.cpu().numpy(), lg.cpu().numpy(), r if kind == 'wide' else dict(r, k=None), kind, g, pr.n_features,
                      '%s %s' % (kind, fam), stats)
            core.close()
    report(front, stats)


# ------------------------------------------------------------------------------------------------------------------ ticks
TICK_NETS = (('std', None), ('keras 1', 96), ('keras 1.3', 64), ('tanh/sigmoid 2', 7), ('tanh/sigmoid 3', 128),
             ('doubling +', 24), ('doubling -', 113))      # ring mode at HP / 16 = 1, 2, 4, 6, 8 and 7 on the wide kernel


def replay(conf, fired, scored, sens=0.5, lvl=3, chunk_bytes=2 * CHUNK):
    """fired [K, S] against OracleTrigger replayed per stream on the GPU's conf [K, S] over the ticks ``scored`` ([S] or
    [K, S] bool) marks; settings per stream or scalar.  Returns each stream's TriggerDetector.activation afterwards."""
    b = lambda v, s: v[s] if np.ndim(v) else v
    scored = np.broadcast_to(scored, conf.shape)
    act = np.zeros(conf.shape[1], np.int64)
    for s in range(conf.shape[1]):
        ks = np.nonzero(scored[:, s])[0]
        det = OracleTrigger(int(b(chunk_bytes, s)), float(b(sens, s)), int(b(lvl, s)))
        assert [bool(det.update(float(conf[k, s]))) for k in ks] == list(fired[ks, s].astype(bool)), s
        act[s] = det.activation
    return act


def activations(core):
    """Bank slot 0's TriggerDetector.activation of every stream, from the exported state records
    (pb_stream_state_header.activation[0], bytes 64 .. 68)."""
    return core.export_streams().cpu().numpy()[:, 64:68].copy().view(np.int32)[:, 0]


def routed_ticks(m, pr, g, S, pcm, sub, routed, modes_and_tags, on_tick):
    """One-model ticks of g on one handle per (mode, tag), all fed pcm.  Routed handles clear bit 0 on the streams ~sub before
    tick ROUTE_AT: those items must come back NaN / NaN / 0 from then on, and their trigger state must stay what it was
    (the exported activation, every tick).  conf == pb_decode(raw) bit for bit; fired, the count and the final activation of
    every stream equal OracleTrigger replayed on the GPU's conf over the ticks each stream was scored.  on_tick(k, hs, sel,
    raws) checks raw."""
    hs = []
    for mode, tag in modes_and_tags:
        sb = m.StreamBatch(g, S, params=pr, chunk_samples=CHUNK)
        sb.core.gru_mode(mode)
        hs.append((tag, sb))
    K = pcm.shape[1] // CHUNK
    conf = np.zeros((len(hs), K, S))
    fired = np.zeros((len(hs), K, S), np.uint8)
    scored = np.ones((K, S), bool)
    held = None
    for k in range(K):
        if routed and k == ROUTE_AT:
            for _, sb in hs:
                sb.set_stream_models(np.where(sub, 1, 0).astype(np.uint8))
            held = [activations(sb.core) for _, sb in hs]
        sel = sub if routed and k >= ROUTE_AT else np.ones(S, bool)
        scored[k] = sel
        c = cuda(pcm[:, k * CHUNK:(k + 1) * CHUNK])
        got = [sb.update(c) for _, sb in hs]
        raws = []
        for j, ((tag, sb), o) in enumerate(zip(hs, got)):
            raw = o['raw'].cpu().numpy().copy()
            conf[j, k], fired[j, k] = o['conf'].cpu().numpy(), o['fired'].cpu().numpy()
            assert np.isnan(raw[~sel]).all() and np.isnan(conf[j, k, ~sel]).all() and not fired[j, k, ~sel].any()
            dec = sb.core.decode(o['raw'][cuda(np.nonzero(sel)[0])]).cpu().numpy()
            assert np.array_equal(dec, conf[j, k, sel]), (tag, k)
            if held is not None:
                assert np.array_equal(activations(sb.core)[~sub], held[j][~sub]), (tag, k)
            raws.append(raw)
        on_tick(k, hs, sel, raws)
    for j, (tag, sb) in enumerate(hs):
        act = replay(conf[j], fired[j], scored)
        assert np.array_equal(activations(sb.core), act), tag
        assert int(sb.count.item()) == int(fired[j].sum())
        if routed:
            print('%s: %d of %d unsubscribed streams held a non-zero trigger state' % (tag, int(np.count_nonzero(held[j][~sub])),
                                                                                   int((~sub).sum())))
        sb.core.close()


@gpu
@pytest.mark.parametrize('front', list(FRONT_ENDS))
def test_one_model_ticks(front):
    """pb_update of one network per family (the std one at the front end's largest H), mode 0 and mode 1 handles fed the same
    audio; every other network routed (bit 0 cleared on streams s % 5 == 2 from tick ROUTE_AT, see routed_ticks).  raw within
    the bounds on the checked ticks' windows."""
    m = _mod()
    pr = params(front)
    F, T = pr.feature_size, pr.n_features
    fi = list(FRONT_ENDS).index(front)
    S = 48
    pcm = audio(S, TICKS * CHUNK, seed=20 + fi)
    sub = np.arange(S) % 5 != 2
    stats = {}
    for i, (fam, H) in enumerate(TICK_NETS):
        if fam.startswith('doubling') and T > 100:                  # h near 2^T leaves float32's range
            continue
        if fam == CHAOTIC[0] and T > CHAOTIC[1]:
            continue
        H = limit_h(F) if H is None else H
        g = FAMILIES[fam](F, H, 400 + i, ACTS[(i + fi) % 4])
        routed = (i + fi) % 2 == 1

        def on_tick(k, hs, sel, raws):
            if k not in CHECKED:
                return
            win = read_windows(hs[0][1].core, pr, S)
            r = refs(weights(g), win[sel], 'wide' if hs[0][0] == 'wide' else None)
            for (kind, _), raw in zip(hs, raws):
                check(raw[sel], None, r if kind == 'wide' else dict(r, k=None), kind, g, T,
                      '%s %s%s' % (kind, fam, ' routed' if routed else ''), stats)

        routed_ticks(m, pr, g, S, pcm, sub, routed, [(mode, kernel_of(F, H, mode)) for mode in modes(F, H)], on_tick)
    report(front + ' ticks', stats)


# ------------------------------------------------------------------------------------------------------------------- banks
def bank_spec(F):
    """(family, H) per slot: fused slots where the front end has them, wide and tiled slots, a doubling slot."""
    spec = [('keras 1', 65), ('std', 17), ('tanh/sigmoid 2', 200), ('keras 1.3', 24), ('std', 128), ('doubling +', 33),
            ('tanh/sigmoid 3', limit_h(F))]
    return [(fam, H, FAMILIES[fam](F, H, 500 + i, ACTS[i % 4])) for i, (fam, H) in enumerate(spec)]


def slot_kind(F, H, use_delta):
    return 'fused' if H <= 24 and F <= 16 and not use_delta else kernel_of(F, H, 0)


@gpu
@pytest.mark.parametrize('front', ['default', 'delta', 'config3', 'f41'])
def test_bank_ticks(front):
    """pb_update_models with seven slots (fused slots where F <= 16), unrouted and routed (random masks), on the same audio;
    slot 2 with per-stream trigger settings.  raw within each slot's kernel bound, fired and counts equal to OracleTrigger on
    the GPU's conf with each stream's settings."""
    m = _mod()
    pr = params(front)
    F, T = pr.feature_size, pr.n_features
    spec = bank_spec(F)
    S = 64
    rs = np.random.RandomState(8)
    masks = rs.randint(0, 128, S).astype(np.uint8)
    sens = rs.uniform(0.2, 0.9, S)
    lvl = rs.randint(0, 6, S).astype(np.int32)
    chunk_bytes = rs.choice([1024, 2 * CHUNK, 9000], S).astype(np.int32)
    arms = []
    for routed in (False, True):
        sb = m.StreamBatch(spec[0][2], S, params=pr, chunk_samples=CHUNK)
        for _, _, g in spec[1:]:
            sb.add_model(g, pr)
        sb.core.set_stream_trigger(2, sens, lvl, chunk_bytes)
        if routed:
            sb.set_stream_models(masks)
        arms.append((routed, sb))
    pcm = audio(S, TICKS * CHUNK, seed=31)
    M = len(spec)
    conf = np.zeros((2, TICKS, M, S))
    fired = np.zeros((2, TICKS, M, S), np.uint8)
    stats = {}
    for k in range(TICKS):
        c = cuda(pcm[:, k * CHUNK:(k + 1) * CHUNK])
        for a, (routed, sb) in enumerate(arms):
            o = sb.update_models(c)
            raw = o['raw'].cpu().numpy()
            conf[a, k], fired[a, k] = o['conf'].cpu().numpy(), o['fired'].cpu().numpy()
            if k not in CHECKED:
                continue
            win = read_windows(sb.core, pr, S)
            for i, (fam, H, g) in enumerate(spec):
                sel = (masks >> i & 1).astype(bool) if routed else np.ones(S, bool)
                assert np.isnan(raw[i, ~sel]).all() and not fired[a, k, i, ~sel].any()
                kind = slot_kind(F, H, pr.use_delta)
                r = refs(weights(g), win[sel], kind if kind != 'tiled' else None)
                check(raw[i, sel], None, r, kind, g, T, '%s %s' % (kind, fam), stats)
    for a, (routed, sb) in enumerate(arms):
        for i in range(M):
            sel = (masks >> i & 1).astype(bool) if routed else np.ones(S, bool)
            if i == 2:
                replay(conf[a, :, i], fired[a, :, i], sel, sens, lvl, chunk_bytes)
            else:
                replay(conf[a, :, i], fired[a, :, i], sel)
        assert np.array_equal(sb.counts.cpu().numpy(), fired[a].sum(axis=(0, 2)))
        sb.core.close()
    report(front + ' bank', stats)


@gpu
@pytest.mark.parametrize('front', ['delta', 'f41'])
def test_ragged_ticks(front):
    """pb_update_ragged of a wide (or tiled) and a tiled network with lengths 1 .. 4 001 that leave n_samples odd: raw within
    the bounds on the windows after each tick."""
    m = _mod()
    pr = params(front)
    F, T = pr.feature_size, pr.n_features
    ga, gb = keras_like(F, 48, 61, 1.0, ACTS[3]), std_model(F, limit_h(F), 62, ACTS[1])
    S = 40
    sb = m.StreamBatch(ga, S, params=pr, chunk_samples=CHUNK)
    sb.add_model(gb, pr)
    rs = np.random.RandomState(9)
    src = audio(S, 30 * 4001, seed=12)
    pos = np.zeros(S, np.int64)
    stats = {}
    for k in range(12):
        lens = rs.randint(1, 4002, S)
        chunks = [src[s, pos[s]:pos[s] + lens[s]] for s in range(S)]
        pos += lens
        offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        o = sb.core.update_ragged(cuda(np.concatenate(chunks)), cuda(offsets))
        raw = o['raw'].cpu().numpy()
        win = read_windows(sb.core, pr, S)
        for i, g in enumerate((ga, gb)):
            kind = kernel_of(F, g.hidden, 0)
            check(raw[i], None, refs(weights(g), win, kind if kind == 'wide' else None), kind, g, T, '%s ragged' % kind, stats)
    assert (pos % 2 == 1).any()
    report(front, stats)
    sb.core.close()


# ------------------------------------------------------------------------------------------------------------------ corpus
@gpu
@pytest.mark.parametrize('front', ['default', 'delta', 'f41', 'd_t73'])
def test_corpus_vs_ticks(front):
    """pb_score_corpus (listener schedule: the predict-mode delta read of input_value) of a wide-eligible slot 0 and a tiled
    slot 1, in both modes: raw within 1e-5 of one stream tick per chunk over the same recordings, within the bounds of the
    float64 GRU on the ticks' windows, and within 1e-4 of the oracle listener end to end once per kernel."""
    m = _mod()
    pr = params(front)
    F, T = pr.feature_size, pr.n_features
    g0, g1 = std_model(F, 100, 71, ACTS[0]), std_model(F, limit_h(F), 72, ACTS[2])
    c, K, S = 1024, 36, 6
    pcm = audio(8, K * c, seed=14)[[0, 1, 2, 3, 5, 7]]
    offsets = np.arange(S + 1, dtype=np.int64) * K * c
    sb = m.StreamBatch(g0, S, params=pr, chunk_samples=c)
    sb.add_model(g1, pr)
    tick_raw = np.zeros((2, S, K), np.float32)
    stats = {}
    for k in range(K):
        o = sb.update_models(cuda(pcm[:, k * c:(k + 1) * c]))
        tick_raw[:, :, k] = o['raw'].cpu().numpy()
        if k % 7 == 6:
            win = read_windows(sb.core, pr, S)
            for i, g in enumerate((g0, g1)):
                kind = kernel_of(F, g.hidden, 0)
                check(tick_raw[i, :, k], None, refs(weights(g), win, kind if kind == 'wide' else None), kind, g, T,
                      '%s ticks' % kind, stats)
    for mode in modes(F, g0.hidden):
        sb.core.gru_mode(mode)
        got = sb.core.score_corpus(cuda(pcm.reshape(-1)), offsets, 'listener', c)
        raw = got['raw'].cpu().numpy().reshape(2, S, K)
        err = float(np.max(np.abs(raw - tick_raw)))
        print('%s mode %d: corpus vs ticks %.2g' % (front, mode, err))
        assert err < 1e-5, (mode, err)
        oraw, _, _ = run_streams(weights(g0), pcm[:2], c, pr=OracleParams(**pr.to_dict()))
        err = float(np.max(np.abs(raw[0, :2] - oraw)))
        print('%s %s: corpus vs oracle listener %.2g' % (front, kernel_of(F, g0.hidden, mode), err))
        assert err < 1e-4
    sb.core.close()
    report(front, stats)


# ---------------------------------------------------------------------------------------------------------------- refusals
@gpu
@pytest.mark.parametrize('kw,H', [(dict(n_mfcc=12), 263), (dict(n_filt=21, n_mfcc=21, use_delta=True), 253)])
def test_tiled_limit_refusals(kw, H):
    """F + 3H = 801: StreamBatch, load_weights and add_model raise NotImplementedError; the bank that refused scores bit for
    bit as a twin that never saw the call; F + 3H = 798 (the largest of this front end) loads and meets the bound.  A handle's
    own F and H are fixed when it is created, so load_weights refuses every network on a handle of H 263 (here F 12) and such
    a handle never holds weights: after the refusal it still has none.  A refused network on a handle that holds weights is
    the add_model case."""
    m = _mod()
    pr = m.ListenerParams(**kw)
    F, T = pr.feature_size, pr.n_features
    assert F + 3 * H == 801
    big = std_model(F, H, 81, ACTS[0])
    with pytest.raises(NotImplementedError, match='too large for the tiled GRU kernel'):
        m.StreamBatch(big, 4, params=pr)
    core = m.PreciseB200(pr, hidden=H)
    with pytest.raises(NotImplementedError, match='too large for the tiled GRU kernel'):
        core.load_weights(big.kernel, big.recurrent, big.bias, big.dense_w, big.dense_b)
    with pytest.raises(Exception, match='has not been called'):
        core.predict(cuda(np.zeros((1, T, F), np.float32)))
    core.close()
    S = 24
    ok = std_model(F, H - 1, 82, ACTS[1])
    a, b = (m.StreamBatch(std_model(F, 40, 83, ACTS[0]), S, params=pr, chunk_samples=CHUNK) for _ in range(2))
    for sb in (a, b):
        sb.add_model(ok, pr)
    pcm = audio(S, 10 * CHUNK, seed=15)
    stats = {}
    for k in range(10):
        if k == 4:
            with pytest.raises(NotImplementedError, match='too large for the tiled GRU kernel'):
                a.add_model(big, pr)
            assert a.core.num_models == 2
        c = cuda(pcm[:, k * CHUNK:(k + 1) * CHUNK])
        oa, ob = a.update_models(c), b.update_models(c)
        for key in ('raw', 'conf', 'fired'):
            assert np.array_equal(oa[key].cpu().numpy(), ob[key].cpu().numpy()), (k, key)
        win = read_windows(a.core, pr, S)
        check(oa['raw'][1].cpu().numpy(), None, refs(weights(ok), win, None), 'tiled', ok, T, 'tiled F+3H 798', stats)
    report(str(kw), stats)
    for sb in (a, b):
        sb.core.close()


# ------------------------------------------------------------------------------------- the default network's CUDA-core scans
@gpu
@pytest.mark.parametrize('fam', ['std', 'keras 1', 'keras 1.3', 'doubling +', 'doubling -'])
def test_default_network_cuda_core(fam):
    """The default network (H 20, F 13, Keras's pair) on gru_warp_kernel (mode 0, <= 8 192 items) and gru_small_kernel
    (mode 1): pb_predict at N 1, 300 and 8 192 (checked every 17th) and one-model ticks, routed from tick ROUTE_AT (the ROUTE
    instantiation of gru_small_kernel; see routed_ticks) and not; bounds with p32 as the yardstick."""
    m = _mod()
    pr = m.ListenerParams()
    g = FAMILIES[fam](13, 20, 91, ACTS[0])
    x_all = front_windows('default')
    rs = np.random.RandomState(2)
    stats = {}
    core = predictor(pr, g)
    for N in (1, 300, 8192):
        x = x_all[rs.randint(0, len(x_all), N)]
        sample = np.arange(0, N, 17)
        r = refs(weights(g), x[sample], None)
        for mode in (0, 1):
            core.gru_mode(mode)
            p, lg = core.predict(cuda(x), want_logit=True)
            check(p.cpu().numpy()[sample], lg.cpu().numpy()[sample], r, None, g, 29, '%s predict' % kernel_of(13, 20, mode, True),
                  stats)
    core.close()
    S = 48
    sub = np.arange(S) % 3 != 1
    pcm = audio(S, TICKS * CHUNK, seed=17)
    for routed in (False, True):
        def on_tick(k, hs, sel, raws):
            r = refs(weights(g), read_windows(hs[0][1].core, pr, S)[sel], None)
            for (tag, _), raw in zip(hs, raws):
                check(raw[sel], None, r, None, g, 29, tag + ' ticks', stats)

        routed_ticks(m, pr, g, S, pcm, sub, routed,
                     [(mode, kernel_of(13, 20, mode, True) + (' routed' if routed else '')) for mode in (0, 1)], on_tick)
    report(fam, stats)
