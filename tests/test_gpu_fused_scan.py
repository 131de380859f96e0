"""The fused family's tensor-core GRU scan (gru_bank.cuh: bank_scan, fp16 x 3) against the float64 GRU, over the shapes,
front ends and weight magnitudes it accepts.

Every pool tick, bank tick, corpus call and large-batch pb_predict of a network with H <= 24, feature_size <= 16 and no
deltas runs bank_scan, except that one-model launches (the default network above 8 192 streams, one-model update_models,
a bank with one fused model) run the same arithmetic on warpgroup MMA in gru_wg_kernel (gru_wg.cuh).  Here only
test_operand_range's 9 000-stream ticks reach gru_wg_kernel; test_gpu_wg_scan.py checks it bit for bit against the
mma.sync kernels and against float64 on every path that reaches it.  The other test files check those paths mostly for bit identity with each other; here each one is
anchored to oracle.gru.gru_forward in float64 on the window the GPU itself scored (read_window after each tick), which
isolates the scan from the MFCC front end, with one end-to-end check per front end against the oracle listeners.

- Shapes: feature sizes 1, 5, 13 and 16 (MFCCs and log-mels), window lengths T = 1, 3, 19, 24, 25, 26, 29, 34, 73 and 281
  (every T mod 4 of the staged rows), hidden sizes 1 .. 24 with partial k8 tiles, all four activation pairs, block and
  warp pool tiles, young windows with leading zero rows, silence and full-scale audio.
- Weight magnitudes: std 0.1, Keras-initialiser-like weights (glorot-uniform kernel, orthogonal recurrent blocks, zero
  bias) at gain 1 and 1.3, and tanh / sigmoid networks at gain 2 and 3.  No trained Precise model ships with the reference
  and none can be fetched, so "trained-like" is an assumption built from Keras's default initialisers.  Bounds: where the
  float32 GRU is within 1e-6 of float64, |raw - p64| < 1e-5; everywhere |raw - p64| <= 2 |p_f16x3 - p64| + 2 |p32 - p64|
  + 1e-6, with p_f16x3 = oracle.gru.gru_forward_f16x3.
- Operand range: networks whose hidden state doubles every step leave fp16's range after 16 steps.  The scan's operand
  split saturates there, so raw, conf and fired stay finite and make the float64 network's saturated decision on every
  path (one-model ticks below and above 8 192 streams, pb_predict in both kernel modes, pool ticks, corpus calls).

-m gpu throughout."""
import numpy as np
import pytest

from oracle import gru as og
from oracle.listener import OracleListener, run_streams
from oracle.params import OracleParams
from oracle.trigger import OracleTrigger

gpu = pytest.mark.gpu
CHUNK = 2048
TICKS = 14                  # 28 672 samples: every window length here fills, and the first ticks score young windows
HIDDEN = (1, 2, 3, 7, 8, 15, 16, 17, 23, 24)
ACTS = (('linear', 'hard_sigmoid'), ('tanh', 'sigmoid'), ('linear', 'sigmoid'), ('tanh', 'hard_sigmoid'))


def _mod():
    import mycroft_precise_b200 as m
    return m


def cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


FRONT_ENDS = {                 # name: ListenerParams arguments (T = n_features, F = feature_size)
    'default': {},                                      # F 13, T 29
    'f16': dict(n_mfcc=16),                             # F 16
    'f5': dict(n_mfcc=5, n_filt=12),                    # F 5
    'f1': dict(n_mfcc=1),                               # F 1
    'mels16': dict(vectorizer=1, n_filt=16, n_mfcc=16), # F 16, log-mels (n_mfcc sizes the oracle listener's rows)
    't1': dict(buffer_t=0.1),
    't3': dict(buffer_t=0.2),
    't19': dict(buffer_t=1.0),
    't24': dict(buffer_t=1.25),
    't25': dict(buffer_t=1.3),
    't26': dict(buffer_t=1.35),
    't34': dict(buffer_t=1.75),
    't73': dict(hop_t=0.02, window_t=0.05),
    't281': dict(hop_t=0.005),
}


def params(name):
    return _mod().ListenerParams(**FRONT_ENDS[name])


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
    """z = 0, r = 1, candidate recurrent block 2 I, candidate bias 1: h_t = 2 h_(t-1) + 1 in every unit, whatever the input
    (h reaches 2^29 - 1 at T = 29, far past fp16's 65 504).  The Dense layer, sign (1e-4 sum(h) / H - 2), decides only once h
    is past about 20 000: prob -> 1 or 0 in float64, and in a scan whose operands saturate (h settles near 262 000).  A scan
    that loses the state there decides otherwise: an inf operand turns the gates' h products into NaN, hard_sigmoid's
    fmaxf turns NaN into r = z = 0, and h restarts from 1 (raw 0.765 for either sign); with a sigmoid recurrent activation
    nothing turns the NaN back into a number."""
    m = _mod()
    rec = np.zeros((H, 3 * H))
    rec[:, 2 * H:] = 2 * np.eye(H)
    bias = np.concatenate([np.full(H, -10.0), np.full(H, 10.0), np.ones(H)])
    g = m.GruModel(np.zeros((F, 3 * H)), rec, bias, np.full(H, 1e-4 * sign / H), -2.0 * sign)
    g.activation, g.recurrent_activation = act
    return g


def grid_models(F):
    """Forty std-0.1 networks: every hidden size of HIDDEN with every activation pair."""
    m = _mod()
    out = []
    for i, (H, act) in enumerate((H, a) for a in ACTS for H in HIDDEN):
        g = m.GruModel.random(F, H, seed=1000 + i, scale=0.1)
        g.activation, g.recurrent_activation = act
        out.append(g)
    return out


def assignment(n_models, seed, block=(0, 1)):
    """Models block[0] and block[1] on 70 and 64 streams (block tiles, staged rows), the others on 1 .. 63 (warp tiles,
    direct loads), three streams on none; streams in random order."""
    sizes = [1 + (11 * i) % 63 for i in range(n_models)]
    sizes[block[0]], sizes[block[1]] = 70, 64
    ids = np.concatenate([np.full(z, k, np.int32) for k, z in enumerate(sizes)] + [np.full(3, -1, np.int32)])
    return np.random.RandomState(seed).permutation(ids).astype(np.int32)


def max_err(got, want):
    """max |got - want| after asserting both are finite: a NaN would otherwise drop out of a running maximum."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert np.all(np.isfinite(got)), 'non-finite output for a window a model scores'
    assert np.all(np.isfinite(want))
    return float(np.max(np.abs(got - want))) if got.size else 0.0


def pool_handle(pr, models, S, assign, warp_only=False):
    m = _mod()
    sb = m.StreamBatch(models[0], S, params=pr, chunk_samples=CHUNK)
    sb.set_pool(len(models))
    for i, g in enumerate(models):
        sb.pool_load(i, g, pr)
    sb.set_stream_pool(assign)
    if warp_only:
        assert sb.core.lib.pb_debug_pool_tiles(sb.core._h, 1) == 0
    return sb


def window(sb, S, F):
    return sb.core.read_window(S).cpu().numpy()[..., :F].astype(np.float32)


def oracle_windows(pr, pcm, chunk):
    """[K, T, F] windows of the oracle listener after each chunk of one recording (Listener.update_vectors)."""
    lis = OracleListener(None, pr)
    out = []
    for k in range(len(pcm) // chunk):
        out.append(lis.update_vectors(pcm[k * chunk:(k + 1) * chunk].astype(np.float32) / 32768.0).copy())
    return np.asarray(out, np.float32).reshape(-1, pr.n_features, lis.mfccs.shape[1])


# ---------------------------------------------------------------------------------------------------------------- shapes
@gpu
@pytest.mark.parametrize('front', list(FRONT_ENDS))
def test_pool_shape_grid(front):
    """A pool of forty networks (H in HIDDEN x four activation pairs) per front end, in block and warp tiles and in warp
    tiles only: raw of every tick finite and within 1e-5 of the float64 GRU on the GPU's own windows; one block-tile model
    end to end against the oracle listeners within 1e-4.  The two block-tile models rotate over the front ends (first H 17
    tanh / sigmoid and H 23 linear / sigmoid), so the staged rows meet many hidden sizes and activation pairs."""
    m = _mod()
    pr = params(front)
    F, T = pr.feature_size, pr.n_features
    models = grid_models(F)
    fi = list(FRONT_ENDS).index(front)
    block = ((17 + 7 * fi) % len(models), (28 + 11 * fi) % len(models))
    assign = assignment(len(models), seed=len(front), block=block)
    S = assign.size
    pcm = audio(S, TICKS * CHUNK, seed=7)
    handles = [pool_handle(pr, models, S, assign), pool_handle(pr, models, S, assign, warp_only=True)]
    ws = [weights(g) for g in models]
    raws = np.zeros((2, TICKS, S), np.float32)
    worst = np.zeros(len(models))
    for k in range(TICKS):
        c = cuda(pcm[:, k * CHUNK:(k + 1) * CHUNK])
        for j, sb in enumerate(handles):
            raws[j, k] = sb.update_pool(c)['raw'].cpu().numpy()
        win = window(handles[0], S, F)
        assert win.shape == (S, T, F)
        for mid, w in enumerate(ws):
            sel = assign == mid
            p64 = og.gru_forward(w, win[sel], np.float64)[0]
            worst[mid] = max(worst[mid], max_err(raws[:, k, sel], p64))
    assert np.isnan(raws[:, :, assign < 0]).all()
    desc = lambda i: 'H %d %s / %s' % (models[i].hidden, models[i].activation, models[i].recurrent_activation)
    print('%s (F %d, T %d): worst |raw - p64| %.3g (%s); block tiles: %s' % (
        front, F, T, worst.max(), desc(worst.argmax()), ', '.join('%s %.3g' % (desc(b), worst[b]) for b in block)))
    assert worst.max() < 1e-5, worst
    # end to end: the first eight streams of the first block-tile model through the oracle listeners
    sids = np.nonzero(assign == block[0])[0][:8]
    oraw, _, _ = run_streams(ws[block[0]], pcm[sids], CHUNK, pr=OracleParams(**pr.to_dict()))
    err = max(max_err(raws[j][:, sids].T, oraw) for j in range(2))
    print('%s: |raw - oracle listener| %.3g' % (front, err))
    assert err < 1e-4
    for sb in handles:
        sb.core.close()


# ------------------------------------------------------------------------------------------------------ other entry points
def bank_of(pr, models, S, chunk=CHUNK):
    m = _mod()
    sb = m.StreamBatch(models[0], S, params=pr, chunk_samples=chunk)
    for g in models[1:]:
        sb.add_model(g, pr)
    return sb


@gpu
@pytest.mark.parametrize('front', ['f16', 't25', 'f5'])
def test_bank_entry_points(front):
    """Unrouted banks of 2 (staged rows), 3 and 8 models (direct ring loads), a routed bank of 3 with compiled-in and run-time
    activations, and update_all's bank and pool rows: raw within 1e-5 of the float64 GRU on the GPU's windows."""
    pr = params(front)
    F = pr.feature_size
    models = grid_models(F)
    pick = [models[i] for i in (9, 13, 3, 36, 27, 18, 6, 24)]      # H 24, 3, 7, 17, 23, 23, 16, 15 over all four pairs
    S = 150
    pcm = audio(S, TICKS * CHUNK, seed=11)
    routed = bank_of(pr, [models[5], models[15], models[8]], S)      # Keras's pair (compiled in), tanh / sigmoid, Keras's
    masks = np.random.RandomState(3).randint(0, 8, S).astype(np.uint8)
    routed.set_stream_models(masks)
    combo = bank_of(pr, pick[:3], S)
    combo.set_pool(4)
    for i, g in enumerate(pick[4:]):
        combo.pool_load(i, g, pr)
    passign = (np.arange(S) % 5 - 1).astype(np.int32)
    combo.set_stream_pool(passign)
    arms = {'bank2': (bank_of(pr, pick[:2], S), pick[:2]), 'bank3': (bank_of(pr, pick[:3], S), pick[:3]),
            'bank8': (bank_of(pr, pick, S), pick), 'routed': (routed, [models[5], models[15], models[8]]),
            'all': (combo, pick[:3])}
    worst = {a: 0.0 for a in arms}
    for k in range(TICKS):
        c = cuda(pcm[:, k * CHUNK:(k + 1) * CHUNK])
        for a, (sb, ms) in arms.items():
            o = (sb.update_all(c) if a == 'all' else sb.update_models(c))['raw'].cpu().numpy()
            win = window(sb, S, F)
            for i, g in enumerate(ms):
                sel = np.ones(S, bool) if a != 'routed' else (masks >> i & 1).astype(bool)
                assert np.isnan(o[i, ~sel]).all()
                p64 = og.gru_forward(weights(g), win[sel], np.float64)[0]
                worst[a] = max(worst[a], max_err(o[i, sel], p64))
            if a == 'all':
                for mid, g in enumerate(pick[4:]):
                    sel = passign == mid
                    p64 = og.gru_forward(weights(g), win[sel], np.float64)[0]
                    worst[a] = max(worst[a], max_err(o[len(ms), sel], p64))
                assert np.isnan(o[len(ms), passign < 0]).all()
    print(front, 'worst |raw - p64|', {a: '%.3g' % v for a, v in worst.items()})
    assert max(worst.values()) < 1e-5, worst
    for sb, _ in arms.values():
        sb.core.close()


@gpu
@pytest.mark.parametrize('front', ['f16', 't25', 'f1'])
def test_corpus_calls(front):
    """score_corpus_pool and score_corpus_pairs (listener schedule) against the float64 GRU on the oracle listener's windows
    of each recording, within 1e-4."""
    m = _mod()
    pr = params(front)
    opr = OracleParams(**pr.to_dict())
    F = pr.feature_size
    models = grid_models(F)
    ids = np.asarray([9, 13, 3, 36, 27], np.int32)
    rs = np.random.RandomState(5)
    recs = [np.clip(rs.randn(16000 * 3 + 77) * s, -32768, 32767).astype(np.int16) for s in (300, 3000, 12000)]
    recs += [np.zeros(20000, np.int16), np.full(20000, -32768, np.int16), np.full(5000, 32767, np.int16)]
    offsets = np.concatenate([[0], np.cumsum([len(r) for r in recs])]).astype(np.int64)
    c = 1024
    h = m.PreciseB200(pr)
    h.set_pool(len(models))
    for i in ids:
        h.pool_load(int(i), models[i], pr)
    wins = [oracle_windows(opr, r, c)[..., :F] for r in recs]
    wo = np.concatenate([[0], np.cumsum([len(w) for w in wins])])
    got = h.score_corpus_pool(cuda(np.concatenate(recs)), offsets, ids, 'listener', c)
    raw = got['raw'].cpu().numpy()
    worst = 0.0
    for row, mid in enumerate(ids):
        for r, w in enumerate(wins):
            if len(w):
                p64 = og.gru_forward(weights(models[mid]), w, np.float64)[0]
                worst = max(worst, max_err(raw[row, wo[r]:wo[r + 1]], p64))
    pm, pr_ = np.asarray([36, 9, 36, 3], np.int32), np.asarray([5, 0, 2, 3], np.int32)
    got = h.score_corpus_pairs(cuda(np.concatenate(recs)), offsets, pm, pr_, 'listener', c)
    raw, P = got['raw'].cpu().numpy(), got['pair_offsets']
    for p, (mid, r) in enumerate(zip(pm, pr_)):
        p64 = og.gru_forward(weights(models[mid]), wins[r], np.float64)[0] if len(wins[r]) else np.zeros(0)
        assert P[p + 1] - P[p] == len(p64)
        if len(p64):
            worst = max(worst, max_err(raw[P[p]:P[p + 1]], p64))
    print('%s: corpus worst |raw - p64| %.3g' % (front, worst))
    assert worst < 1e-4
    h.close()


# ------------------------------------------------------------------------------------------------------- weight magnitudes
FAMILIES = {
    'std 0.1': lambda F, H, seed, act: _random(F, H, seed, act),
    'keras gain 1': lambda F, H, seed, act: keras_like(F, H, seed, 1.0, act),
    'keras gain 1.3': lambda F, H, seed, act: keras_like(F, H, seed, 1.3, act),
    'tanh/sigmoid gain 2': lambda F, H, seed, act: keras_like(F, H, seed, 2.0, ACTS[1]),
    'tanh/sigmoid gain 3': lambda F, H, seed, act: keras_like(F, H, seed, 3.0, ACTS[1]),
}


def _random(F, H, seed, act):
    g = _mod().GruModel.random(F, H, seed=seed, scale=0.1)
    g.activation, g.recurrent_activation = act
    return g


def bound_check(got, x, w, tag, stats):
    """The two bounds of the module docstring on probabilities; returns nothing, records the worst values under ``tag``."""
    p64 = og.gru_forward(w, x, np.float64)[0]
    p32 = og.gru_forward(w, x, np.float32)[0].astype(np.float64)
    pf = og.gru_forward_f16x3(w, x)[0].astype(np.float64)
    e, e32, ef = np.abs(got - p64), np.abs(p32 - p64), np.abs(pf - p64)
    assert np.all(np.isfinite(got)), tag
    tight = e32 < 1e-6
    assert np.all(e[tight] < 1e-5), (tag, float(e[tight].max()))
    assert np.all(e <= 2 * ef + 2 * e32 + 1e-6), (tag, float(np.max(e - 2 * ef - 2 * e32)))
    s = stats.setdefault(tag, np.zeros(3))
    stats[tag] = np.maximum(s, [e.max(), ef.max(), e32.max()])


@gpu
@pytest.mark.parametrize('front', ['default', 'f16', 't25'])
def test_weight_magnitudes(front):
    """Five weight families, twelve networks each (H 8, 17, 20 and 24, three seeds, Keras's pair unless the family fixes
    tanh / sigmoid), in one pool over noise, silence and full-scale streams: the bounds of the module docstring on every tick.
    On the default front end also pb_predict's logit (gru_mode 2, the default network's tensor-core scan) on the same
    windows, under the same rules applied to logits: where the float32 logit is within 4e-6 of float64, |logit - l64|
    < 5e-5 (test_gpu_parity's logit bound); everywhere |logit - l64| <= 2 |l_f16x3 - l64| + 2 |l32 - l64| + 4e-6 max(1,
    |l64|).  The logit constants are the probability rule's over sigmoid's slope of at most 1/4, and relative past |logit|
    1, where float32 rounding of the logit itself grows with it.  Prints the worst |raw - p64|, |p_f16x3 - p64| and
    |p32 - p64|."""
    m = _mod()
    pr = params(front)
    F = pr.feature_size
    spec = []
    for fam, make in FAMILIES.items():
        for i, H in enumerate((8, 17, 20, 24) * 3):
            spec.append((fam, make(F, H, 200 + i, ACTS[0])))
    models = [g for _, g in spec]
    S = 8 * len(models)
    assign = np.random.RandomState(1).permutation(np.repeat(np.arange(len(models), dtype=np.int32), 8))
    sb = pool_handle(pr, models, S, assign)
    pcm = audio(S, TICKS * CHUNK, seed=13)
    stats = {}
    wins = []
    for k in range(TICKS):
        raw = sb.update_pool(cuda(pcm[:, k * CHUNK:(k + 1) * CHUNK]))['raw'].cpu().numpy().astype(np.float64)
        win = window(sb, S, F)
        if k >= TICKS - 4:
            wins.append(win)
        for mid, (fam, g) in enumerate(spec):
            sel = assign == mid
            bound_check(raw[sel], win[sel], weights(g), fam, stats)
    for fam, (e, ef, e32) in stats.items():
        print('%s %s: |raw - p64| %.3g, |p_f16x3 - p64| %.3g, |p32 - p64| %.3g' % (front, fam, e, ef, e32))
    sb.core.close()
    if front != 'default':
        return
    x = np.concatenate(wins)
    lstats = {}
    for fam, g in spec:
        if g.hidden != 20 or (g.activation, g.recurrent_activation) != ACTS[0]:     # the default network's shape
            continue
        core = m.PreciseB200(pr)
        core.gru_mode(2)
        core.load_weights(g.kernel, g.recurrent, g.bias, g.dense_w, g.dense_b)
        _, lg = core.predict(cuda(x), want_logit=True)
        lg = lg.cpu().numpy().astype(np.float64)
        w = weights(g)
        l64 = og.gru_forward(w, x, np.float64)[1]
        l32 = og.gru_forward(w, x, np.float32)[1].astype(np.float64)
        lf = og.gru_forward_f16x3(w, x)[1].astype(np.float64)
        assert np.all(np.isfinite(lg)), fam
        e, e32, ef = np.abs(lg - l64), np.abs(l32 - l64), np.abs(lf - l64)
        tight = e32 < 4e-6
        assert np.all(e[tight] < 5e-5), (fam, float(e[tight].max()))
        slack = 4e-6 * np.maximum(1.0, np.abs(l64))
        assert np.all(e <= 2 * ef + 2 * e32 + slack), (fam, float(np.max(e - 2 * ef - 2 * e32 - slack)))
        s = lstats.setdefault(fam, np.zeros(3))
        lstats[fam] = np.maximum(s, [e.max(), ef.max(), e32.max()])
        core.close()
    for fam, (e, ef, e32) in lstats.items():
        print('pb_predict logit %s: |logit - l64| %.3g, |l_f16x3 - l64| %.3g, |l32 - l64| %.3g' % (fam, e, ef, e32))
    assert len(lstats) == 3


# ---------------------------------------------------------------------------------------------------------- operand range
def replay(conf, fired, sens=0.5, lvl=3, chunk=CHUNK):
    """fired [K, S] against OracleTrigger replayed per stream on the GPU's conf [K, S]."""
    for s in range(conf.shape[1]):
        det = OracleTrigger(2 * chunk, sens, lvl)
        assert [bool(det.update(float(c))) for c in conf[:, s]] == list(fired[:, s].astype(bool)), s


@gpu
@pytest.mark.parametrize('sign', [1.0, -1.0])
def test_operand_range(sign):
    """Doubling networks (|h| past fp16's range) on every path: raw, conf and fired finite, equal across paths and equal to
    the float64 network's saturated decision within 1e-5; fired and the counts match OracleTrigger on the GPU's conf."""
    m = _mod()
    pr = m.ListenerParams()
    want = 1.0 if sign > 0 else 0.0
    d20, d16 = doubling(13, 20, sign), doubling(13, 16, sign)
    K = 6
    outs = {}
    for S in (300, 9000):                     # gru_warp_kernel (fp32) and gru_wg_kernel (fp16 x 3)
        pcm = audio(64, K * 1024, seed=S)
        pcm = np.tile(pcm, (S // 64 + 1, 1))[:S].copy()
        sb = m.StreamBatch(d20, S)
        raw, conf, fired = [], [], []
        for k in range(K):
            o = sb.update(cuda(pcm[:, k * 1024:(k + 1) * 1024]))
            raw.append(o['raw'].cpu().numpy().copy())
            conf.append(o['conf'].cpu().numpy().copy())
            fired.append(o['fired'].cpu().numpy().copy())
        win = window(sb, S, 13)
        p64 = og.gru_forward(weights(d20), win[::97], np.float64)[0]
        assert np.all(np.abs(p64 - want) < 1e-5)
        raw, conf, fired = np.asarray(raw), np.asarray(conf), np.asarray(fired)
        assert np.all(np.isfinite(raw)) and np.all(np.isfinite(conf)), S
        assert np.all(np.abs(raw - want) < 1e-5) and np.all((conf > 0.5) == (sign > 0)), S
        replay(conf[:, ::41], fired[:, ::41], chunk=1024)
        assert int(sb.count.item()) == int(fired.sum())
        outs['update %d' % S] = raw
        sb.core.close()
    # pb_predict, both kernel modes, on the last windows of the large tick
    core = m.PreciseB200(pr, max_streams=1)
    core.load_weights(d20.kernel, d20.recurrent, d20.bias, d20.dense_w, d20.dense_b)
    x = (np.random.RandomState(2).randn(9000, 29, 13) * 10).astype(np.float32)
    for mode in (1, 2):
        core.gru_mode(mode)
        p, lg = core.predict(cuda(x), want_logit=True)
        p, lg = p.cpu().numpy(), lg.cpu().numpy()
        assert np.all(np.isfinite(lg)) and np.all(np.abs(p - want) < 1e-5), mode
        assert np.all(np.sign(lg) == sign), mode
        outs['predict %d' % mode] = p
    core.close()
    # a pool tick (H 16 and 20 with Keras's pair, H 16 linear / sigmoid) and the pool's corpus call
    S = 200
    pool = pool_handle(pr, [d16, d20, doubling(13, 16, sign, ACTS[2])], S, (np.arange(S) % 3).astype(np.int32))
    pcm = audio(S, TICKS * CHUNK, seed=4)
    raw, conf, fired = [], [], []
    for k in range(TICKS):
        o = pool.update_pool(cuda(pcm[:, k * CHUNK:(k + 1) * CHUNK]))
        raw.append(o['raw'].cpu().numpy().copy())
        conf.append(o['conf'].cpu().numpy().copy())
        fired.append(o['fired'].cpu().numpy().copy())
    raw, conf, fired = np.asarray(raw), np.asarray(conf), np.asarray(fired)
    assert np.all(np.isfinite(raw)) and np.all(np.abs(raw - want) < 1e-5)
    assert np.all(np.isfinite(conf)) and np.all((conf > 0.5) == (sign > 0))
    replay(conf, fired)
    assert int(pool.pool_count.item()) == int(fired.sum())
    outs['pool'] = raw
    recs = [pcm[0, :30000], pcm[4, :20000], pcm[5, :9000]]
    offsets = np.concatenate([[0], np.cumsum([len(r) for r in recs])]).astype(np.int64)
    got = pool.core.score_corpus_pool(cuda(np.concatenate(recs)), offsets, np.asarray([0, 1, 2], np.int32), 'listener', 1024)
    craw, cconf, cfired = (got[k].cpu().numpy() for k in ('raw', 'conf', 'fired'))
    assert np.all(np.isfinite(craw)) and np.all(np.abs(craw - want) < 1e-5)
    assert np.all(np.isfinite(cconf)) and np.all((cconf > 0.5) == (sign > 0))
    wo = np.concatenate([[0], np.cumsum([len(r) // 1024 for r in recs])])
    for row in range(3):
        for i in range(len(recs)):
            det = OracleTrigger(2 * 1024, 0.5, 3)
            assert [bool(det.update(float(c))) for c in cconf[row, wo[i]:wo[i + 1]]] == list(cfired[row, wo[i]:wo[i + 1]].astype(bool))
    outs['corpus'] = craw
    pool.core.close()
    vals = {k: np.unique(v) for k, v in outs.items()}
    print('sign %+d: distinct raw per path %s' % (sign, vals))
    allv = np.concatenate(list(vals.values()))
    assert allv.max() - allv.min() < 1e-5                 # fp32 paths reach 0.0 where the saturated scan gives 3e-11
