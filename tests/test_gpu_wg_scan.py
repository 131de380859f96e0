"""The one-model fused-family scan on warpgroup MMA (gru_wg_kernel, gru_wg.cuh) against the mma.sync scans bit for bit and
against the float64 GRU, on every call path that reaches it.

gru_wg_kernel adds each accumulator's products in bank_scan's order, so it must give the same bits as the mma.sync kernels
(gru_bank_kernel, gru_bank_routed_kernel) on the same windows.  That is also a library invariant: a routed handle scores
fused models on gru_bank_routed_kernel and an unrouted one-model handle on gru_wg_kernel, and streams exported from one
and imported into the other continue bit for bit only if the two scans agree.  Which launches reach it (api.cu:
launch_gru_kernels, launch_bank_nm, score_bank, score_bank_routed, pb_score_corpus), and the mma.sync twin each is compared with:

| Route                                                       | gru_wg_kernel<RING, KERAS_ACT> | mma.sync twin on the same inputs |
|-------------------------------------------------------------|--------------------------------|----------------------------------|
| default network: update and one-model update_ragged above   | <true, true>                   | the routed handle's update_models |
| 8 192 streams, or under gru_mode(2) at any n; also on a      |                                | (gru_bank_routed_kernel<true>); a bank [d, d]'s update_models |
| routed handle (the epilogue's route mask)                   |                                | and update_ragged (gru_bank_kernel<2, true, false>) |
| any fused network: one-model unrouted update_models, any n  | <true, true> for Keras's pair, | the same model on a routed handle, every stream subscribed |
|                                                             | else <true, false>             | (gru_bank_routed_kernel<KERAS_ACT>); a bank [g, g] (gru_bank_kernel<2, true, false>) |
| default network: pb_predict above 8 192 items or under      | <false, true>                  | the twin tick's raw on the windows read back with read_window; |
| gru_mode(2); one-model score_corpus above 8 192 windows     |                                | a corpus call on the bank [d, d] (gru_bank_kernel<2, false, false>) |
| score_corpus on a bank with exactly one fused model beside  | <false, KERAS_ACT of g>        | the same corpus on the bank [g, g, wide] (row 0 against rows 0 and 1) |
| non-fused (wide / tiled) ones                               |                                |                                  |

set_stream_models makes a handle routed for good, and fused models on a routed handle always run gru_bank_routed_kernel, so
an all-ones mask is an mma.sync twin.  A one-model update_ragged runs pb_update's network path (score_model0), so a
non-default fused network there, as on update, pb_predict or a one-model corpus, runs gru_wide_kernel, not gru_wg_kernel;
those paths are not counted here.  A handle's activation pair is fixed when it is
created (load_weights replaces weights only), so the two tick instantiations are reached by networks of either pair rather
than by reloading slot 0.

- Dispatch guard: torch.profiler shows each route launching its gru_wg_kernel instantiation (all four) and each twin an
  mma.sync kernel, so a later dispatch change cannot turn the twin tests into self-comparisons.
- Bit twins on ticks: test_gpu_fused_scan's forty networks (H 1 .. 24 with partial k8 tiles x four activation pairs)
  rotate over its fourteen front ends (F 1, 5, 13, 16, log-mels; T 1 .. 281, every T mod 4 of the staged rows) and over
  n = 1, 15, 16, 17, 63, 64, 65, 129 (and 8 257 = 129 x 64 + 1): warps wholly past n still run wgmma.  Ticks are full
  and permuted subsets; some streams restart, so young windows (leading zero rows) are scored beside full ones, and
  the chunk is not a multiple of the hop, so window starts move through the ring.  raw and conf bits, fired and counts of
  the wgmma handle must equal its routed twin's and both rows of its [g, g] bank's.
- Default network: update and update_ragged, unrouted and routed (some streams unsubscribed), against the routed twin's
  update_models and a bank [d, d] at n = 9 000 and 8 193, and under gru_mode(2) at n = 1, 63, 65 and 300, with a weight
  reload mid-run; pb_predict on the
  windows each tick scored must give the twin's raw bit for bit (N = 9 000, 8 193 and, under gru_mode(2), 1 .. 300).
- Corpus calls: the default network alone above 8 192 windows against the bank [d, d], and for every activation pair a
  bank [g, wide] against [g, g, wide]: raw, conf, fired and activations bit for bit.
- Float64: every route is also anchored to oracle.gru.gru_forward in float64 on the GPU's own windows (read_window after
  each tick; pb_predict's input), with test_gpu_fused_scan's rules: |raw - p64| < 1e-5 where float32 is within 1e-6 of
  float64, and everywhere |raw - p64| <= 2 |p_f16x3 - p64| + 2 |p32 - p64| + 1e-6 (for the weight families over each
  tick's worst outputs, a measured exception: see call_bound); the corpus calls, whose windows the
  GPU does not expose, within 1e-4 of float64 on the oracle listener's windows.  Weight families: std 0.1, Keras-like at
  gain 1 and 1.3, tanh / sigmoid at gain 2 and 3, and doubling networks at H 16, 17 and 24 (units 16..23 are the
  zero-padded k16) whose raw must be float64's saturated decision.

-m gpu throughout."""
import re

import numpy as np
import pytest

torch = pytest.importorskip('torch')

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='needs a CUDA GPU (H100)')]

from oracle import gru as og                                                             # noqa: E402
from test_gpu_fused_scan import (ACTS, FAMILIES, FRONT_ENDS, HIDDEN, audio, bound_check, cuda, doubling,  # noqa: E402
                                 grid_models, keras_like, max_err, oracle_windows, params, weights)
from oracle.params import OracleParams                                                   # noqa: E402

SIZES = (1, 15, 16, 17, 63, 64, 65, 129)
BIG = 129 * 64 + 1                # 8 257 streams: one stream in the last warpgroup
TICKS = 14


def _mod():
    import mycroft_precise_b200 as m
    return m


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view({4: np.uint32, 8: np.uint64, 1: np.uint8}[a.dtype.itemsize])


def same(tag, got, want):
    """got and want bit for bit; on a difference, where and how many."""
    g, w = bits(got), bits(want)
    assert g.shape == w.shape, (tag, g.shape, w.shape)
    bad = np.nonzero(g != w)
    assert not bad[0].size, '%s: %d of %d differ, first at %s: %r vs %r' % (
        tag, bad[0].size, g.size, tuple(int(b[0]) for b in bad), np.asarray(got)[tuple(b[0] for b in bad)],
        np.asarray(want)[tuple(b[0] for b in bad)])


def host(o):
    return {k: v.cpu().numpy().copy() for k, v in o.items()}


def chunk_of(pr):
    """A tick length that is not a multiple of the hop (ticks release alternating frame counts, so window starts move
    through the ring) and fills a window in about ten ticks."""
    return pr.hop_samples * (pr.n_features // 10 + 1) + pr.hop_samples // 3


def win_of(core, ids_t, F):
    return core.read_window(ids=ids_t).cpu().numpy()[..., :F]


# ------------------------------------------------------------------------------------------------------------ tick twins
class Twins:
    """Network g on three handles fed the same ticks: 'wg' (one model, unrouted: gru_wg_kernel<true, KERAS_ACT>), 'routed'
    (the same model, every stream subscribed: gru_bank_routed_kernel<KERAS_ACT>) and 'bank' ([g, g]: gru_bank_kernel<2,
    true, false>, both rows)."""

    def __init__(self, pr, g, S, chunk):
        m = _mod()
        self.wg = m.StreamBatch(g, S, params=pr, chunk_samples=chunk)
        self.routed = m.StreamBatch(g, S, params=pr, chunk_samples=chunk)
        self.routed.set_stream_models(np.ones(S, np.uint8))
        self.bank = m.StreamBatch(g, S, params=pr, chunk_samples=chunk)
        self.bank.add_model(g, pr)
        self.handles = (self.wg, self.routed, self.bank)

    def tick(self, tag, pcm, ids=None):
        """One tick on every handle; asserts the twins' bits and returns the wgmma handle's raw [n]."""
        outs = [host(sb.update_models(pcm, ids)) for sb in self.handles]
        a, r, b = outs
        for key in ('raw', 'conf', 'fired'):
            same('%s %s routed' % (tag, key), a[key][0], r[key][0])
            same('%s %s bank row 0' % (tag, key), a[key][0], b[key][0])
            same('%s %s bank row 1' % (tag, key), a[key][0], b[key][1])
        c = [sb.counts.cpu().numpy() for sb in self.handles]
        assert c[0][0] == c[1][0] == c[2][0] == c[2][1], (tag, c)
        return a['raw'][0]

    def clear(self, ids_t):
        for sb in self.handles:
            sb.clear(ids_t)

    def close(self):
        for sb in self.handles:
            sb.core.close()


class Source:
    """Audio of S streams: test_gpu_fused_scan.audio for up to 256 streams; above that its 64 streams repeated, every
    seventh copy read 123 samples further on."""

    def __init__(self, S, n, seed):
        self.big = S > 256
        self.pcm = audio(64 if self.big else S, n + 123, seed)

    def take(self, ids, pos, lens):
        if not self.big:
            return [self.pcm[s, p:p + n] for s, p, n in zip(ids, pos, lens)]
        return [self.pcm[s % 64, p + 123 * (s % 7 == 0):p + 123 * (s % 7 == 0) + n] for s, p, n in zip(ids, pos, lens)]


def run_twins(pr, g, S, seed, check, ticks=TICKS):
    """Ticks of network g over S streams on Twins: full, permuted, permuted subsets, and a restart of some streams halfway.
    check(k, raw, win) gets the wgmma raw of each tick and the windows it scored."""
    F = pr.feature_size
    chunk = chunk_of(pr)
    rs = np.random.RandomState(seed)
    src = Source(S, 2 * ticks * chunk, seed)
    pos = np.zeros(S, np.int64)
    tw = Twins(pr, g, S, chunk)
    for k in range(ticks):
        if k == ticks // 2:
            cl = rs.permutation(S)[:max(1, S // 3)].astype(np.int32)
            tw.clear(cuda(cl))
        kind = k % 3
        ids = np.arange(S, dtype=np.int32) if kind == 0 else rs.permutation(S).astype(np.int32)
        if kind == 1:
            ids = ids[:rs.randint(1, S + 1)]
        ids_t = cuda(ids)
        tag = 'H %d %s/%s S %d tick %d' % (g.hidden, g.activation, g.recurrent_activation, S, k)
        pcm = np.stack(src.take(ids, pos[ids], np.full(len(ids), chunk)))
        raw = tw.tick(tag, cuda(pcm), ids_t)
        pos[ids] += chunk
        check(k, raw, win_of(tw.wg.core, ids_t, F))
    tw.close()


@pytest.mark.parametrize('front', list(FRONT_ENDS))
def test_tick_twins_grid(front):
    """Ten of the forty grid networks per front end (all forty over four front ends in turn), each on its own stream count
    of SIZES: the bit twins of every tick, and raw within 1e-5 of the float64 GRU on the GPU's windows."""
    pr = params(front)
    F = pr.feature_size
    fi = list(FRONT_ENDS).index(front)
    models = grid_models(F)
    worst = 0.0
    for j, g in enumerate(models):
        if (j + fi) % 4:
            continue
        w = weights(g)
        S = SIZES[(j // 4 + fi) % len(SIZES)]

        def check(k, raw, win):
            nonlocal worst
            worst = max(worst, max_err(raw, og.gru_forward(w, win, np.float64)[0]))

        run_twins(pr, g, S, seed=100 * fi + j, check=check)
    print('%s: worst |raw - p64| %.3g' % (front, worst))
    assert worst < 1e-5


@pytest.mark.parametrize('front,j', [('f16', 26), ('t25', 9), ('f1', 3)])
def test_tick_twins_large(front, j):
    """8 257 streams (one stream in the last warpgroup) with grid network j: the bit twins of every tick and raw within 1e-5
    of float64 on a strided sample of the windows."""
    pr = params(front)
    g = grid_models(pr.feature_size)[j]
    w = weights(g)
    worst = 0.0

    def check(k, raw, win):
        nonlocal worst
        sel = np.r_[0:len(raw):37, len(raw) - 1]
        worst = max(worst, max_err(raw[sel], og.gru_forward(w, win[sel], np.float64)[0]))

    run_twins(pr, g, BIG, seed=j, check=check, ticks=10)
    print('%s H %d %s/%s, %d streams: worst |raw - p64| %.3g' % (front, g.hidden, g.activation, g.recurrent_activation,
                                                               BIG, worst))
    assert worst < 1e-5


@pytest.mark.parametrize('front', ['default', 'f16', 't25'])
def test_tick_twins_weight_families(front):
    """Five weight families at H 8, 17 and 24 (Keras's pair, or tanh / sigmoid where the family fixes it), and doubling
    networks at H 16, 17 and 24 of either sign (Keras's pair and linear / sigmoid), on one-model ticks of 65 streams: the bit
    twins; the bounds of the module docstring on every tick, the relative one over the tick's worst outputs (call_bound); doubling raw finite and float64's saturated decision within
    1e-5.  Prints the worst |raw - p64|, |p_f16x3 - p64| and |p32 - p64| per family."""
    pr = params(front)
    F = pr.feature_size
    stats = {}
    for fi, (fam, make) in enumerate(FAMILIES.items()):
        for i, H in enumerate((8, 17, 24)):
            g = make(F, H, 300 + 3 * fi + i, ACTS[0])
            w = weights(g)
            run_twins(pr, g, 65, seed=fi * 3 + i,
                      check=lambda k, raw, win: call_bound(raw.astype(np.float64), win, w, fam, stats))
    dworst = 0.0
    for i, H in enumerate((16, 17, 24)):
        for sign in (1.0, -1.0):
            g = doubling(F, H, sign, ACTS[0] if i % 2 == 0 else ACTS[2])
            want = 1.0 if sign > 0 else 0.0

            def check(k, raw, win):
                nonlocal dworst
                assert np.all(np.abs(og.gru_forward(weights(g), win, np.float64)[0] - want) < 1e-5)
                dworst = max(dworst, max_err(raw, np.full(len(raw), want)))

            run_twins(pr, g, 65, seed=50 + i, check=check)
    for fam, (e, ef, e32) in stats.items():
        print('%s %s: |raw - p64| %.3g, |p_f16x3 - p64| %.3g, |p32 - p64| %.3g' % (front, fam, e, ef, e32))
    print('%s doubling: |raw - decision| %.3g' % (front, dworst))
    assert dworst < 1e-5


def call_bound(got, x, w, tag, stats):
    """bound_check with its relative rule over one call's outputs: max |raw - p64| <= 2 max |p_f16x3 - p64| + 2 max |p32 -
    p64| + 1e-6, as test_gpu_wide_scan applies it.  Measured on the H100: per output, Keras-like gain 1.3 networks at H 8 .. 24
    exceed the rule by up to 4.8e-6 on single outputs whose own f16x3 and float32 errors are small by chance, with the
    wgmma and mma.sync scans bit-identical there, so the excess belongs to the fp16 x 3 design both share."""
    p64 = og.gru_forward(w, x, np.float64)[0]
    p32 = og.gru_forward(w, x, np.float32)[0].astype(np.float64)
    pf = og.gru_forward_f16x3(w, x)[0].astype(np.float64)
    e, e32, ef = np.abs(got - p64), np.abs(p32 - p64), np.abs(pf - p64)
    assert np.all(np.isfinite(got)), tag
    tight = e32 < 1e-6
    assert np.all(e[tight] < 1e-5), (tag, float(e[tight].max()))
    assert e.max() <= 2 * ef.max() + 2 * e32.max() + 1e-6, (tag, float(e.max()), float(ef.max()), float(e32.max()))
    s = stats.setdefault(tag, np.zeros(3))
    stats[tag] = np.maximum(s, [e.max(), ef.max(), e32.max()])


# ------------------------------------------------------------------------------------------------------- default network
@pytest.mark.parametrize('S', [9000, 8193, 1, 63, 65, 300])
def test_default_network_twins(S):
    """The default network's update and update_ragged, unrouted and routed with about a fifth of the streams unsubscribed
    (gru_wg_kernel<true, true>), against a bank [d, d]'s update_models and update_ragged (gru_bank_kernel<2, true, false>,
    both rows until the reload, which replaces slot 0 only) and, on uniform ticks, the routed twin's update_models (gru_bank_routed_kernel<true>), bit for bit: raw, conf,
    fired and counts; pb_predict on the windows each tick scored equal to the bank's raw.  Above 8 192 streams in the
    automatic mode, below it under gru_mode(2).  Weights are reloaded halfway (std 0.1, then Keras-like at gain 1.3).  Every
    tick's raw and every pb_predict logit are anchored to float64 with the module docstring's rules; below 8 192 streams
    2 400-sample ticks (3 frames, prime to the 32-row ring) and ragged ones move full windows' starts through every ring
    slot (from 63 streams on)."""
    m = _mod()
    large = S > 8192
    mode = 0 if large else 2
    K, chunk = (10, 2400) if large else (50, 2400)
    d1 = m.GruModel.random(13, 20, seed=8, scale=0.1)
    d1.dense_b = 2.0
    d2 = keras_like(13, 20, 9, 1.3)
    rs = np.random.RandomState(S)
    masks = np.where(rs.rand(S) < 0.2, 0, 1).astype(np.uint8)
    masks[0] = 1
    arms = []
    for a in ('unrouted', 'routed', 'twin', 'bank'):
        sb = m.StreamBatch(d1, S, chunk_samples=chunk)
        sb.core.gru_mode(mode)
        if a in ('routed', 'twin'):
            sb.set_stream_models(masks if a == 'routed' else np.ones(S, np.uint8))
        if a == 'bank':
            sb.add_model(d1)
        arms.append(sb)
    un, ro, tw, bk = arms
    pred = m.PreciseB200(max_streams=1)
    pred.load_weights(d1.kernel, d1.recurrent, d1.bias, d1.dense_w, d1.dense_b)
    pred.gru_mode(mode)
    src = Source(S, 2 * K * chunk, seed=S)
    n_samples = np.zeros(S, np.int64)
    pos = np.zeros(S, np.int64)
    starts, young, ragged = set(), 0, 0
    stats, lstats = {}, {}
    g = d1
    for k in range(K):
        if k == K // 2:
            g = d2
            for core in [sb.core for sb in arms] + [pred]:
                core.load_weights(g.kernel, g.recurrent, g.bias, g.dense_w, g.dense_b)
        if k == 3:                                                  # restart a quarter of the streams
            cl = np.sort(rs.permutation(S)[:max(1, S // 4)]).astype(np.int32)
            for sb in arms:
                sb.clear(cuda(cl))
            n_samples[cl] = 0
        ids = rs.permutation(S).astype(np.int32)
        if k % 3 == 1:
            ids = ids[:rs.randint(8193 if large else 1, S + 1)]
        ids_t = cuda(ids)
        tag = 'S %d tick %d' % (S, k)
        if k % 5 == 2:                                              # ragged: 1 .. 2 chunks per item
            lens = rs.randint(1, 2 * chunk + 1, len(ids))
            pcm = cuda(np.concatenate(src.take(ids, pos[ids], lens)))
            offsets = cuda(np.concatenate([[0], np.cumsum(lens)]).astype(np.int64))
            o_un, o_ro, o_tw, o_bk = (host(sb.update_ragged(pcm, offsets, ids_t)) for sb in arms)
            o_tw = None                                              # a one-model ragged tick runs update's scan
            ragged += 1
        else:
            lens = np.full(len(ids), chunk)
            pcm = cuda(np.stack(src.take(ids, pos[ids], lens)))
            o_un, o_ro = host(un.update(pcm, ids_t)), host(ro.update(pcm, ids_t))
            o_tw, o_bk = host(tw.update_models(pcm, ids_t)), host(bk.update_models(pcm, ids_t))
        pos[ids] += lens
        n_samples[ids] += lens
        sub = masks[ids] == 1
        for key in ('raw', 'conf', 'fired'):
            want = o_bk[key][0]
            if g is d1:                                             # load_weights replaces slot 0 only
                same('%s %s bank row 1' % (tag, key), o_bk[key][1], want)
            same('%s %s unrouted' % (tag, key), o_un[key].reshape(-1), want)
            same('%s %s routed' % (tag, key), o_ro[key].reshape(-1)[sub], want[sub])
            if o_tw is not None:
                same('%s %s routed twin' % (tag, key), o_tw[key][0], want)
        assert np.isnan(o_ro['raw'].reshape(-1)[~sub]).all() and not o_ro['fired'].reshape(-1)[~sub].any(), tag
        fires = [int(sb.count.item()) + int(sb.counts[0].item()) for sb in (un, tw, bk)]
        assert len(set(fires)) == 1, (tag, fires)
        win_t = bk.core.read_window(ids=ids_t)
        p, lg = pred.predict(win_t, want_logit=True)
        same('%s pb_predict' % tag, p.cpu().numpy(), o_bk['raw'][0])
        win = win_t.cpu().numpy()
        same('%s windows' % tag, win_of(un.core, ids_t, 13), win)
        sel = slice(None) if not large else np.r_[0:len(ids):29, len(ids) - 1]
        fam = 'std 0.1' if g is d1 else 'keras gain 1.3'
        bound_check(o_un['raw'].reshape(-1)[sel].astype(np.float64), win[sel], weights(g), fam, stats)
        logit_check(lg.cpu().numpy()[sel], win[sel], weights(g), fam, lstats)
        ns = n_samples[ids]
        released = np.where(ns >= 1600, (ns - 1600) // 800 + 1, 0)
        full = released >= 29
        starts.update(((released[full] - 29) % 32).tolist())
        young += int(np.count_nonzero(~full & (released > 0)))
    for c in arms:
        c.core.close()
    pred.close()
    for fam, (e, ef, e32) in stats.items():
        print('S %d update %s: |raw - p64| %.3g, |p_f16x3 - p64| %.3g, |p32 - p64| %.3g' % (S, fam, e, ef, e32))
    for fam, (e, ef, e32) in lstats.items():
        print('S %d pb_predict logit %s: |logit - l64| %.3g, |l_f16x3 - l64| %.3g, |l32 - l64| %.3g' % (S, fam, e, ef, e32))
    assert young > 0 and ragged > 0
    if 1 < S < 8193:                      # one stream's window starts step by its frames per tick
        assert starts == set(range(32)), sorted(set(range(32)) - starts)


def logit_check(lg, x, w, tag, stats):
    """test_gpu_fused_scan.test_weight_magnitudes's logit rule: where the float32 logit is within 4e-6 of float64, |logit -
    l64| < 5e-5; everywhere |logit - l64| <= 2 |l_f16x3 - l64| + 2 |l32 - l64| + 4e-6 max(1, |l64|)."""
    l64 = og.gru_forward(w, x, np.float64)[1]
    l32 = og.gru_forward(w, x, np.float32)[1].astype(np.float64)
    lf = og.gru_forward_f16x3(w, x)[1].astype(np.float64)
    assert np.all(np.isfinite(lg)), tag
    e, e32, ef = np.abs(lg - l64), np.abs(l32 - l64), np.abs(lf - l64)
    tight = e32 < 4e-6
    assert np.all(e[tight] < 5e-5), (tag, float(e[tight].max()))
    slack = 4e-6 * np.maximum(1.0, np.abs(l64))
    assert np.all(e <= 2 * ef + 2 * e32 + slack), (tag, float(np.max(e - 2 * ef - 2 * e32 - slack)))
    s = stats.setdefault(tag, np.zeros(3))
    stats[tag] = np.maximum(s, [e.max(), ef.max(), e32.max()])


# ---------------------------------------------------------------------------------------------------------------- corpus
def recordings(seed, n_long, long_len):
    """Noise at four levels, silence, +-full scale, a square wave, a recording shorter than a window, and n_long long
    noise recordings."""
    rs = np.random.RandomState(seed)
    recs = [np.clip(rs.randn(16000 * 2 + 77) * s, -32768, 32767).astype(np.int16) for s in (30, 300, 3000, 12000)]
    recs += [np.zeros(20000, np.int16), np.full(20000, 32767, np.int16), np.full(9000, -32768, np.int16),
             np.where((np.arange(30011) // 37) % 2, 32767, -32767).astype(np.int16), np.full(1000, 500, np.int16)]
    recs += [np.clip(rs.randn(long_len + 113 * i) * 3000, -32768, 32767).astype(np.int16) for i in range(n_long)]
    return recs


def corpus_handle(pr, models):
    m = _mod()
    g = models[0]
    h = m.PreciseB200(pr, hidden=g.hidden, activation=g.activation, recurrent_activation=g.recurrent_activation)
    h.load_weights(g.kernel, g.recurrent, g.bias, g.dense_w, g.dense_b)
    for x in models[1:]:
        h.add_model(x, pr)
    return h


def corpus_twins(pr, g, one, twin, rows, recs, c, anchor):
    """score_corpus of bank ``one`` (row 0 on gru_wg_kernel) and bank ``twin``: each of one's rows bit for bit equal to
    twin's rows[i] (a list of rows per row); row 0 within 1e-4 of float64 on the oracle listener's windows of recordings
    ``anchor`` (g: row 0's network).  Returns that error and W."""
    pcm = cuda(np.concatenate(recs))
    offsets = np.concatenate([[0], np.cumsum([len(r) for r in recs])]).astype(np.int64)
    a = host({k: v for k, v in one.score_corpus(pcm, offsets, 'listener', c).items() if v is not None})
    b = host({k: v for k, v in twin.score_corpus(pcm, offsets, 'listener', c).items() if v is not None})
    for i, want in enumerate(rows):
        for j in want:
            for key in ('raw', 'conf', 'fired', 'activations'):
                same('corpus %s row %d vs twin row %d' % (key, i, j), a[key][i], b[key][j])
    W = a['raw'].shape[1]
    wo = np.concatenate([[0], np.cumsum([one.corpus_windows(len(r), 'listener', c) for r in recs])])
    F = pr.feature_size
    opr = OracleParams(**pr.to_dict())
    err = 0.0
    for r in anchor:
        win = oracle_windows(opr, recs[r], c)[..., :F]
        assert len(win) == wo[r + 1] - wo[r]
        if len(win):
            err = max(err, max_err(a['raw'][0, wo[r]:wo[r + 1]], og.gru_forward(weights(g), win, np.float64)[0]))
    return err, W


def test_default_corpus_twins():
    """The default network alone over more than 8 192 windows (gru_wg_kernel<false, true>) against the bank [d, d]
    (gru_bank_kernel<2, false, false>): raw, conf, fired and activations bit for bit; raw within 1e-4 of float64 on the
    oracle listener's windows of the short recordings."""
    m = _mod()
    pr = m.ListenerParams()
    d = keras_like(13, 20, 21, 1.0)
    d.dense_b = 1.0
    one, twin = corpus_handle(pr, [d]), corpus_handle(pr, [d, d])
    recs = recordings(3, 20, 460000)
    err, W = corpus_twins(pr, d, one, twin, [[0, 1]], recs, 1024, anchor=range(9))
    print('default network corpus, %d windows: |raw - p64| %.3g' % (W, err))
    assert W > 8192
    assert err < 1e-4
    one.close()
    twin.close()


@pytest.mark.parametrize('act,front', [(ACTS[0], 'f16'), (ACTS[1], 't25'), (ACTS[2], 'f5'), (ACTS[3], 'default')])
def test_mixed_corpus_twins(act, front):
    """A bank [g, wide] (gru_wg_kernel<false, KERAS_ACT of g> beside gru_wide_kernel) against [g, g, wide]
    (gru_bank_kernel<2, false, false>): g's row bit for bit equal to both fused rows, the wide row to the wide row; g's raw
    within 1e-4 of float64 on the oracle listener's windows."""
    m = _mod()
    pr = params(front)
    F = pr.feature_size
    g = grid_models(F)[ACTS.index(act) * len(HIDDEN) + HIDDEN.index(17)]          # units 16..23: the zero-padded k16
    wide = m.GruModel.random(F, 40, seed=7, scale=0.1)
    one, twin = corpus_handle(pr, [g, wide]), corpus_handle(pr, [g, g, wide])
    err, W = corpus_twins(pr, g, one, twin, [[0, 1], [2]], recordings(4, 2, 50000), 1024, anchor=range(11))
    print('%s H %d %s/%s [g, wide] corpus, %d windows: |raw - p64| %.3g' % (front, g.hidden, act[0], act[1], W, err))
    assert err < 1e-4
    one.close()
    twin.close()


# ------------------------------------------------------------------------------------------------------- dispatch guard
def kernels(fn):
    """Names of the GRU kernels fn launches."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {e.key for e in prof.key_averages() if 'gru_' in e.key}


WG = re.compile(r'gru_wg_kernel<(true|false), (true|false)>')
MMA = re.compile(r'gru_bank(_routed)?_kernel<')


def test_dispatch_guard():
    """Each route of the module docstring launches its gru_wg_kernel instantiation and nothing else of the GRU kernels, and
    each twin launches an mma.sync kernel (gru_bank_kernel or gru_bank_routed_kernel) and no gru_wg_kernel; all four
    instantiations appear."""
    m = _mod()
    pr = m.ListenerParams()
    d = m.GruModel.random(13, 20, seed=1, scale=0.1)
    g = m.GruModel.random(13, 17, seed=2, scale=0.1)
    g.activation, g.recurrent_activation = ACTS[1]
    wide = m.GruModel.random(13, 40, seed=3, scale=0.1)
    S, chunk = 65, 1024
    pcm = cuda(audio(S, chunk, seed=1))
    dn = m.StreamBatch(d, S)
    dn.core.gru_mode(2)
    dr = m.StreamBatch(d, S)
    dr.set_stream_models(np.ones(S, np.uint8))
    dr.core.gru_mode(2)
    big = m.StreamBatch(d, 9000)
    bigp = cuda(np.stack(Source(9000, chunk, seed=2).take(range(9000), np.zeros(9000, int), np.full(9000, chunk))))
    tw = Twins(pr, g, S, chunk)
    bb = m.StreamBatch(d, S)
    bb.add_model(d)
    lens = np.random.RandomState(1).randint(1, 2 * chunk + 1, S)
    rpcm1 = cuda(np.concatenate(Source(S, 2 * chunk, seed=3).take(range(S), np.zeros(S, int), lens)))
    roff = cuda(np.concatenate([[0], np.cumsum(lens)]).astype(np.int64))
    pred = m.PreciseB200(max_streams=1)
    pred.load_weights(d.kernel, d.recurrent, d.bias, d.dense_w, d.dense_b)
    pred.gru_mode(2)
    x = cuda(np.random.RandomState(0).randn(65, 29, 13).astype(np.float32))
    recs = recordings(5, 0, 0)
    rpcm = cuda(np.concatenate(recs))
    offsets = np.concatenate([[0], np.cumsum([len(r) for r in recs])]).astype(np.int64)
    dd = corpus_handle(pr, [d, d])
    gw, ggw = corpus_handle(pr, [g, wide]), corpus_handle(pr, [g, g, wide])
    corpus = lambda h: lambda: h.score_corpus(rpcm, offsets, 'listener', 1024)
    routes = {                        # name: (call, its gru_wg_kernel instantiation or None for a twin)
        'update above 8 192': (lambda: big.update(bigp), ('true', 'true')),
        'update, gru_mode(2)': (lambda: dn.update(pcm), ('true', 'true')),
        'routed update, gru_mode(2)': (lambda: dr.update(pcm), ('true', 'true')),
        'routed update_models (twin)': (lambda: dr.update_models(pcm), None),
        'one-model update_models, tanh/sigmoid': (lambda: tw.wg.update_models(pcm), ('true', 'false')),
        'one-model update_models, Keras': (lambda: dn.update_models(pcm), ('true', 'true')),
        'routed update_models, tanh/sigmoid (twin)': (lambda: tw.routed.update_models(pcm), None),
        'bank [g, g] (twin)': (lambda: tw.bank.update_models(pcm), None),
        'update_ragged, gru_mode(2)': (lambda: dn.update_ragged(rpcm1, roff), ('true', 'true')),
        'bank [d, d] update_ragged (twin)': (lambda: bb.update_ragged(rpcm1, roff), None),
        'pb_predict, gru_mode(2)': (lambda: pred.predict(x), ('false', 'true')),
        'corpus [d, d] (twin)': (corpus(dd), None),
        'corpus [g, wide]': (corpus(gw), ('false', 'false')),
        'corpus [g, g, wide] (twin)': (corpus(ggw), None),
    }
    seen = set()
    for name, (fn, want) in routes.items():
        fn()                                                       # warm-up
        names = kernels(fn)
        wg = {WG.search(k).groups() for k in names if WG.search(k)}
        mma = {k for k in names if MMA.search(k)}
        print('%s: %s' % (name, sorted(names)))
        if want is None:
            assert mma and not wg, (name, names)
        else:
            assert wg == {want} and not mma, (name, names)
            seen.add(want)
    assert seen == {('true', 'true'), ('true', 'false'), ('false', 'true'), ('false', 'false')}, seen
    for h in (dn.core, dr.core, big.core, bb.core, pred, dd, gw, ggw):
        h.close()
    tw.close()
