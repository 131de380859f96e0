"""-m gpu: CUDA path (through the C ABI) vs the oracle on the same seeded inputs.

Tolerances
  * MFCC rows: abs 2e-4 on realistic-amplitude audio (the kernel computes in fp32, the reference in
    float64); exact -36.0437 / ln 512 rows on the reference's own all-zero / constant test signals.
  * GRU output on identical inputs: abs 1e-5 (BASELINE.json north_star), vs the fp32 AND fp64 oracle.  The fused
    family's fp16 x 3 scan (H <= 24, feature_size <= 16, no deltas: pools, banks, corpus calls and the default network above
    8 192 streams) is anchored to float64 over its shapes, front ends, weight magnitudes and operand range in
    test_gpu_fused_scan.py, with oracle.gru.gru_forward_f16x3 bounding what larger weights may cost; its one-model form on
    warpgroup MMA (gru_wg_kernel) is checked bit for bit against the mma.sync kernels in test_gpu_wg_scan.py.  The other networks'
    scans (gru_wide_kernel's 3 x TF32, gru_tiled_kernel) and the default network's CUDA-core scans (gru_warp_kernel,
    gru_small_kernel) are anchored the same way in test_gpu_wide_scan.py, with oracle.gru.gru_forward_tf32x3 as the wide
    kernel's reference.
  * decode: bit-identical conf for the same raw, except that the LUT index may move by one bin
    when CUDA's log() and libm's differ in the last ulp (rate reported, must be < 0.2 %).
  * trigger / count: exact.
"""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')

from oracle import gru as og                      # noqa: E402
from oracle import mfcc as om                     # noqa: E402
from oracle.decoder import OracleDecoder          # noqa: E402
from oracle.listener import run_streams, OracleListener   # noqa: E402
from oracle.params import OracleParams            # noqa: E402
from oracle.trigger import OracleTrigger          # noqa: E402


def _mod():
    import mycroft_precise_b200 as m
    return m


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def noise(S, L, seed=0, sigma=3000):
    rs = np.random.RandomState(seed)
    return np.clip(rs.randn(S, L) * sigma, -32768, 32767).astype(np.int16)


def oracle_pr(pr):
    return OracleParams(**pr.to_dict())


def oracle_mfcc(pcm_i16, pr):
    return np.stack([om.vectorize_raw(r.astype(np.float32) / 32768.0, oracle_pr(pr)) for r in pcm_i16])


@pytest.fixture(scope='module')
def core():
    m = _mod()
    c = m.PreciseB200(max_streams=64)
    yield c
    c.close()


# ------------------------------------------------------------------------------------------ tables
def test_filterbank_bit_equal(core):
    assert np.array_equal(core.filterbank(), om.filterbank(16000, 20, 257))


def test_cdf_tables(core):
    d = OracleDecoder(((6, 4),), 0.2)
    cd, lo, hi = core.cdf()
    assert (lo, hi) == (d.min_out, d.max_out) and len(cd) == 6400
    assert np.array_equal(cd, d.cd)                # numpy-built table uploaded by the host
    m = _mod()
    import ctypes as C
    from mycroft_precise_b200.core import make_config, get_lib, check
    cfg = make_config(m.ListenerParams())
    h = C.c_void_p()
    check(get_lib().pb_create(C.byref(cfg), C.byref(h)))
    raw = np.zeros(6400)
    get_lib().pb_get_cdf(h, raw.ctypes.data_as(C.c_void_p), 6400, None, None)
    get_lib().pb_destroy(h)
    assert np.max(np.abs(raw - d.cd)) < 1e-14      # libm-built table inside the library


# ------------------------------------------------------------------------------------------ K1
def test_mfcc_batch_noise(core):
    pcm = noise(37, 24000, seed=1)
    got = core.mfcc(cuda(pcm)).cpu().numpy()
    want = oracle_mfcc(pcm, core.params)
    assert got.shape == want.shape == (37, 29, 13)
    err = np.max(np.abs(got - want))
    print('mfcc max abs err', err)
    assert err < 2e-4


def test_generic_kernels_on_default_geometry():
    """The any-alignment kernels (mfcc_kernels.cuh) must agree with the warp-autonomous fast kernels
    (mfcc_fast.cuh) that normally serve the default geometry."""
    m = _mod()
    pcm = noise(21, 24000, seed=31)
    a = m.PreciseB200(max_streams=32)
    b = m.PreciseB200(max_streams=32)
    b.force_generic(True)
    ma, mb = a.mfcc(cuda(pcm)).cpu().numpy(), b.mfcc(cuda(pcm)).cpu().numpy()
    want = oracle_mfcc(pcm, a.params)
    assert np.max(np.abs(ma - want)) < 2e-4 and np.max(np.abs(mb - want)) < 2e-4
    assert np.max(np.abs(ma - mb)) < 1e-4
    for k in range(23):
        c = cuda(pcm[:, k * 1024:(k + 1) * 1024])
        a.update_vectors(c)
        b.update_vectors(c)
        wa, wb = a.read_window(21).cpu().numpy(), b.read_window(21).cpu().numpy()
        assert np.max(np.abs(wa - wb)) < 1e-4
    assert np.abs(wa).max() > 1
    a.close(); b.close()


def test_mfcc_lengths_and_ragged_tail(core):
    for L in (1600, 1601, 2399, 2400, 3333, 9999):
        pcm = noise(3, L, seed=L)
        got = core.mfcc(cuda(pcm)).cpu().numpy()
        want = oracle_mfcc(pcm, core.params)
        assert got.shape == want.shape
        assert np.max(np.abs(got - want)) < 2e-4
    assert core.mfcc(cuda(noise(2, 1599))).shape == (2, 0, 13)
    with pytest.raises(ValueError):
        core.mfcc(torch.zeros((1, 0), dtype=torch.int16, device='cuda'))


def test_mfcc_reference_test_signals(core):
    z = core.mfcc(torch.zeros((1, 1600), dtype=torch.int16, device='cuda')).cpu().numpy()[0, 0]
    assert abs(z[0] - (-36.04365338911715)) < 1e-5 and np.all(np.abs(z[1:]) < 1e-5)
    ones = torch.ones((1, 1600), dtype=torch.float32, device='cuda')          # the reference's 1.0 signal
    o = core.mfcc(ones).cpu().numpy()[0, 0]
    assert abs(o[0] - np.log(512.0)) < 1e-5 and np.all(np.abs(o[1:]) < 1e-5)
    dc = torch.full((1, 1600), 32767, dtype=torch.int16, device='cuda')
    d = core.mfcc(dc).cpu().numpy()[0, 0]
    want = om.mfcc_spec(np.full(1600, 32767 / 32768.0), 16000, 1600, 800, 512, 20, 13)[0]
    assert np.max(np.abs(d - want)) < 1e-5


def test_mfcc_tone_and_quiet(core):
    t = np.arange(24000)
    tone = (12000 * np.sin(2 * np.pi * 440.0 * t / 16000)).astype(np.int16)[None]
    quiet = noise(1, 24000, seed=5, sigma=20)
    for pcm, tol in ((tone, 5e-3), (quiet, 2e-4)):
        got = core.mfcc(cuda(pcm)).cpu().numpy()
        want = oracle_mfcc(pcm, core.params)
        err = np.max(np.abs(got - want))
        print('err', err)
        assert err < tol


def test_mfcc_f32_input(core):
    rs = np.random.RandomState(2)
    a = (rs.randn(5, 8000) * 0.1).astype(np.float32)
    got = core.mfcc(cuda(a)).cpu().numpy()
    want = np.stack([om.vectorize_raw(r, oracle_pr(core.params)) for r in a])
    assert np.max(np.abs(got - want)) < 2e-4
    odd = a[:, 1:7000]                                   # misaligned rows: scalar load path
    got = core.mfcc(cuda(odd)).cpu().numpy()
    want = np.stack([om.vectorize_raw(r, oracle_pr(core.params)) for r in odd])
    assert np.max(np.abs(got - want)) < 2e-4


def test_mfcc_linearity_property_large(core):
    """Full-size property check: scaling the PCM by 2 adds ln 4 to c0 and leaves c1.. unchanged."""
    pcm = noise(4096, 8000, seed=7, sigma=2000)
    a = core.mfcc(cuda(pcm))
    b = core.mfcc(cuda((pcm.astype(np.int32) * 2).astype(np.int16)))
    d = (b - a).cpu().numpy()
    assert np.max(np.abs(d[..., 0] - np.log(4.0))) < 1e-4
    assert np.max(np.abs(d[..., 1:])) < 1e-4


# ------------------------------------------------------------------------------------------ K2
@pytest.mark.parametrize('scale', [0.1, 0.3])
def test_predict_small_path(core, scale):
    w = og.GruWeights.random(13, 20, seed=3, scale=scale)
    core.load_weights(w.kernel, w.recurrent, w.bias, w.dense_w, w.dense_b)
    x = (np.random.RandomState(4).randn(1000, 29, 13) * 3).astype(np.float32)
    p, lg = core.predict(cuda(x), want_logit=True)
    p, lg = p.cpu().numpy(), lg.cpu().numpy()
    p32, l32 = og.gru_forward(w, x, np.float32)
    p64, l64 = og.gru_forward(w, x, np.float64)
    print('prob err vs f32 %.3g vs f64 %.3g ; logit rel err %.3g' % (
        np.max(np.abs(p - p32)), np.max(np.abs(p - p64)), np.max(np.abs(lg - l64) / (1 + np.abs(l64)))))
    if scale == 0.1:
        # well-conditioned recurrence (what a trained model looks like): the north-star tolerance
        assert np.max(np.abs(p - p32)) < 1e-5 and np.max(np.abs(p - p64)) < 1e-5
        assert np.max(np.abs(lg - l64) / (1 + np.abs(l64))) < 1e-4
    else:
        # 0.3-scaled random weights make the linear-activation recurrence expansive (spectral radius
        # > 1): fp32 round-off is amplified ~1e4x, and the fp32 ORACLE itself is that far from the fp64
        # oracle.  The kernel must not be worse than the fp32 oracle's own conditioning error.
        ref = np.abs(p32 - p64)
        assert np.max(ref) > 1e-4                       # documents the ill-conditioning
        assert np.max(np.abs(p - p64)) < 4 * np.max(ref) + 1e-5
        assert np.median(np.abs(p - p64)) < 1e-5


@pytest.mark.parametrize('mode', [0, 1, 2])
def test_default_network_kernel_variants(core, mode):
    """warp-per-stream (auto, small n), thread-per-stream CUDA-core (1) and tensor-core fp16 x 3 (2, gru_wg_kernel) kernels."""
    w = og.GruWeights.random(13, 20, seed=11, scale=0.1)
    core.load_weights(w.kernel, w.recurrent, w.bias, w.dense_w, w.dense_b)
    core.gru_mode(mode)
    try:
        for N in (1, 31, 33, 777, 9000):
            x = (np.random.RandomState(N).randn(N, 29, 13) * 3).astype(np.float32)
            p, lg = core.predict(cuda(x), want_logit=True)
            p, lg = p.cpu().numpy(), lg.cpu().numpy()
            sel = slice(None) if N < 2000 else slice(0, None, 7)
            p64, l64 = og.gru_forward(w, x[sel], np.float64)
            err, lerr = np.max(np.abs(p[sel] - p64)), np.max(np.abs(lg[sel] - l64))
            print('mode', mode, 'N', N, 'prob err %.3g logit err %.3g' % (err, lerr))
            assert err < 1e-5 and lerr < 5e-5
    finally:
        core.gru_mode(0)


def test_stream_tick_kernel_variants_agree():
    m = _mod()
    S, K, chunk = 300, 34, 1024
    pcm = noise(S, K * chunk, seed=21)
    model = m.GruModel.random(13, 20, seed=6, scale=0.1)
    model.dense_b = 3.0                                   # pushes the confidence over the trigger threshold
    outs = []
    for mode in (0, 1, 2):
        sb = m.StreamBatch(model, S, chunk_samples=chunk)
        sb.core.gru_mode(mode)
        raws, fired = [], []
        for k in range(K):
            o = sb.update(cuda(pcm[:, k * chunk:(k + 1) * chunk]))
            raws.append(o['raw'].cpu().numpy().copy()); fired.append(o['fired'].cpu().numpy().copy())
        outs.append((np.array(raws), np.array(fired), int(sb.count.item())))
        sb.core.close()
    for r, f, c in outs[1:]:
        assert np.max(np.abs(r - outs[0][0])) < 1e-5
    assert outs[0][2] == outs[0][1].sum() > 0
    # a conf within rounding of the threshold may flip a trigger between variants; allow a handful
    assert all(abs(o[2] - outs[0][2]) <= 3 for o in outs[1:])


def test_large_batch_tensor_core_scan():
    """n > 8192 streams: the tensor-core scan (gru_wg_kernel) vs the CUDA-core kernel, including a weight reload and a
    small-batch tick in between.  A one-model update_models arm goes through the same sequence and must score bit for bit
    like update's scan: a window's score does not depend on the ticks before it.  Both arms run gru_wg_kernel, so that
    comparison is wgmma against itself; test_gpu_wg_scan.py compares it with the mma.sync kernels."""
    m = _mod()
    S, K, chunk = 9000, 36, 1024
    pcm = noise(64, K * chunk, seed=33)
    pcm = np.tile(pcm, (S // 64 + 1, 1))[:S].copy()
    pcm[::7] = np.roll(pcm[::7], 123, axis=1)
    model = m.GruModel.random(13, 20, seed=8, scale=0.1)
    model.dense_b = 3.0

    def run(mode):
        """mode 0 (automatic) / 1 (CUDA cores) through update, or 'bank' through update_models: raw [K][S], detections."""
        sb = m.StreamBatch(model, S, chunk_samples=chunk)
        if mode == 'bank':
            tick = lambda c, ids=None: sb.update_models(c, ids)['raw'][0]
        else:
            sb.core.gru_mode(mode)
            tick = lambda c, ids=None: sb.update(c, ids)['raw']
        raws = []
        for k in range(K):
            if k == 20:                                              # reload weights mid-stream
                sb.core.load_weights(model.kernel, model.recurrent, model.bias, model.dense_w, model.dense_b)
            if k == 25:                                              # a small tick for a few streams (warp-per-stream kernel in update)
                r5 = tick(cuda(pcm[:5, k * chunk:(k + 1) * chunk]), torch.arange(5, dtype=torch.int32, device='cuda')).cpu().numpy()
                r = tick(cuda(pcm[5:, k * chunk:(k + 1) * chunk]), torch.arange(5, S, dtype=torch.int32, device='cuda')).cpu().numpy()
                raws.append(np.concatenate([r5, r]))
                continue
            raws.append(tick(cuda(pcm[:, k * chunk:(k + 1) * chunk])).cpu().numpy())
        count = int(sb.counts[0].item()) if mode == 'bank' else int(sb.count.item())
        sb.core.close()
        return np.array(raws), count

    ref = run(1)
    res = [run(0), run('bank')]
    for r, c in res:
        assert np.max(np.abs(r - ref[0])) < 1e-5
        assert c > 0 and abs(c - ref[1]) <= 3
    a, b = res[0][0].copy(), res[1][0].copy()
    a[25, :5] = b[25, :5] = 0                                        # the 5-stream tick: warp-per-stream kernel in update only
    assert np.array_equal(a, b)
    print('max |raw - CUDA-core kernel|: %.3g' % np.max(np.abs(res[0][0] - ref[0])))


def _generic_case(pr_kw, H, act='linear', ract='hard_sigmoid', N=200, seed=5, mode=0):
    m = _mod()
    pr = m.ListenerParams(**pr_kw)
    c = m.PreciseB200(pr, hidden=H, max_streams=8, activation=act, recurrent_activation=ract)
    F = c.feature_size
    w = og.GruWeights.random(F, H, seed=seed, scale=0.1 / np.sqrt(max(H, 20) / 20.0))   # contractive recurrence
    w.activation, w.recurrent_activation = act, ract
    c.load_weights(w.kernel, w.recurrent, w.bias, w.dense_w, w.dense_b)
    c.gru_mode(mode)
    x = (np.random.RandomState(seed).randn(N, pr.n_features, F) * 2).astype(np.float32)
    p = c.predict(cuda(x)).cpu().numpy()
    p64 = og.gru_forward(w, x, np.float64)[0]
    c.close()
    return np.max(np.abs(p - p64))


@pytest.mark.parametrize('H,kw,act,ract', [
    (32, {}, 'linear', 'hard_sigmoid'),
    (128, dict(n_filt=40, n_mfcc=40), 'linear', 'hard_sigmoid'),     # BASELINE config 3
    (20, dict(use_delta=True), 'linear', 'hard_sigmoid'),
    (20, {}, 'tanh', 'sigmoid'),
    (7, dict(n_mfcc=5), 'tanh', 'hard_sigmoid'),
])
@pytest.mark.parametrize('mode', [0, 1])
def test_predict_tiled_path(H, kw, act, ract, mode):
    """mode 0: automatic choice, mode 1: CUDA-core tiled kernel."""
    err = _generic_case(kw, H, act, ract, mode=mode, N=333)
    print('generic GRU err', err)
    assert err < 1e-5


def test_predict_edge_sizes(core):
    w = og.GruWeights.random(13, 20, seed=3, scale=0.1)
    core.load_weights(w.kernel, w.recurrent, w.bias, w.dense_w, w.dense_b)
    assert core.predict(torch.zeros((0, 29, 13), device='cuda')).shape == (0,)
    for N in (1, 127, 129):
        x = (np.random.RandomState(N).randn(N, 29, 13)).astype(np.float32)
        p = core.predict(cuda(x)).cpu().numpy()
        assert np.max(np.abs(p - og.gru_forward(w, x, np.float64)[0])) < 1e-5
    with pytest.raises(ValueError):
        core.predict(torch.zeros((2, 28, 13), device='cuda'))


# ------------------------------------------------------------------------------------------ K3
def _neighbour_values(d, r):
    """Confidences of the LUT bins next to the one the oracle picks for raw output r."""
    i = d.index(r)
    out = []
    for j in (i - 1, i + 1):
        if 0 <= j < len(d.cd):
            cp = d.cd[j]
            out.append(0.5 * cp / d.center if cp < d.center else 0.5 + 0.5 * (cp - d.center) / (1 - d.center))
    return out


@pytest.mark.parametrize('case', range(5))
@pytest.mark.parametrize('legacy', [False, True], ids=['asigmoid_f32', 'asigmoid_f64'])
def test_decode_vs_reference_golden(golden_dir, case, legacy):
    """pb_decode against values produced by the reference's ThresholdDecoder itself for all DECODER_CASES
    (multi-Gaussian, centre 0.5 / 0.7, std 0 -> out_range 0).  Default mode: the decoder was fed np.float32 scalars
    (what Runner.run returns; `1 / x - 1` in float32 under this image's NumPy) -> dec32_*; decode_legacy_f64: python
    floats (= NumPy 1.16 promotion) -> dec_*."""
    import os
    import sys
    sys.path.insert(0, golden_dir)
    from cases import DECODER_CASES
    m = _mod()
    cfg, center = DECODER_CASES[case]
    pr = m.ListenerParams(threshold_config=cfg, threshold_center=center)
    core = m.PreciseB200(pr, decode_legacy_f64=legacy)
    g = np.load(os.path.join(golden_dir, 'decoder_golden.npz'))
    raws = g['raws']
    got = core.decode(cuda(raws)).cpu().numpy()
    want = g['dec_%d' % case] if legacy else g['dec32_%d' % case]
    d = OracleDecoder(cfg, center)
    exact = got == want
    print('decode case %d legacy=%s: %d / %d bit-identical' % (case, legacy, exact.sum(), len(raws)))
    assert exact.mean() > 0.998                           # libm log vs CUDA log: an ulp can move a value across a bin edge
    for r, a in zip(raws[~exact], got[~exact]):           # the rest: neighbouring LUT bin
        assert any(a == c for c in _neighbour_values(d, float(r) if legacy else r))
    core.close()


# ------------------------------------------------------------------------------------------ stateful
def _run_gpu_streams(m, model, pcm, chunk, pr=None, sens=0.5, lvl=3, host=False, pinned=False):
    S = pcm.shape[0]
    K = pcm.shape[1] // chunk
    sb = m.StreamBatch(model, S, params=pr, chunk_samples=chunk, sensitivity=sens, trigger_level=lvl)
    raw = np.zeros((S, K), np.float32)
    conf = np.zeros((S, K))
    fired = np.zeros((S, K), bool)
    wins = []
    counts = 0
    for k in range(K):
        c = np.ascontiguousarray(pcm[:, k * chunk:(k + 1) * chunk])
        if host and pinned:
            from mycroft_precise_b200.core import pinned_empty, pinned_free
            pc, p0 = pinned_empty(c.shape, np.int16); pc[:] = c
            r, p1 = pinned_empty((S,), np.float32); cf, p2 = pinned_empty((S,), np.float64); f, p3 = pinned_empty((S,), np.uint8)
            counts += sb.update_host(pc, cf, r, f)
            raw[:, k], conf[:, k], fired[:, k] = r, cf, f.astype(bool)
            for p in (p0, p1, p2, p3):
                pinned_free(p)
        elif host:
            r = np.zeros(S, np.float32); cf = np.zeros(S); f = np.zeros(S, np.uint8)
            counts += sb.update_host(c, cf, r, f)
            raw[:, k], conf[:, k], fired[:, k] = r, cf, f.astype(bool)
        else:
            out = sb.update(cuda(c))
            raw[:, k] = out['raw'].cpu().numpy()
            conf[:, k] = out['conf'].cpu().numpy()
            fired[:, k] = out['fired'].cpu().numpy().astype(bool)
        wins.append(sb.core.read_window(S).cpu().numpy())
    if not host:
        counts = int(sb.count.item())
    sb.core.close()
    return raw, conf, fired, np.array(wins), counts


def _oracle_windows(pcm, chunk, pr):
    S, K = pcm.shape[0], pcm.shape[1] // chunk
    w = og.GruWeights.random(pr.n_mfcc if not hasattr(pr, 'feature_size') else 13, 20)
    wins = np.zeros((K, S, pr.n_features, pr.n_mfcc))
    for s in range(S):
        lis = OracleListener(w, pr)
        for k in range(K):
            wins[k, s] = lis.update_vectors(pcm[s, k * chunk:(k + 1) * chunk].astype(np.float32) / 32768.0)
    return wins


@pytest.mark.parametrize('chunk', [1024, 512, 800, 2000, 334, 333])
def test_stream_state_machine(chunk):
    """Window contents, raw, conf, fired after every tick vs S independent oracle Listeners."""
    m = _mod()
    S, K = 7, max(12, 30000 // chunk)
    pcm = noise(S, K * chunk, seed=chunk)
    pcm[5] = 0
    pcm[6] = 32767
    model = m.GruModel.random(13, 20, seed=0, scale=0.1)
    raw, conf, fired, wins, count = _run_gpu_streams(m, model, pcm, chunk, sens=0.8, lvl=1)
    opr = OracleParams()
    owins = _oracle_windows(pcm, chunk, opr)
    werr = np.max(np.abs(wins - owins))
    print('window err', werr)
    assert werr < 2e-4
    w = og.GruWeights(model.kernel, model.recurrent, model.bias, model.dense_w, model.dense_b)
    # GRU on the GPU's own windows: identical inputs -> 1e-5
    p64 = og.gru_forward(w, wins.reshape(-1, 29, 13), np.float64)[0].reshape(K, S).T
    assert np.max(np.abs(raw - p64)) < 1e-5
    # end to end vs oracle listeners
    oraw, oconf, ofired = run_streams(w, pcm, chunk, sensitivity=0.8, trigger_level=1)
    assert np.max(np.abs(raw - oraw)) < 1e-4
    # decode of the GPU raw: exact up to a neighbouring bin
    d = OracleDecoder(opr.threshold_config, opr.threshold_center)
    dconf = np.vectorize(lambda r: d.decode(float(r)))(raw)
    neq = conf != dconf
    assert neq.mean() < 0.01
    step = np.max(np.abs(np.diff(d.cd))) * 2.5
    assert np.max(np.abs(conf - dconf)) <= step
    # trigger on the GPU conf: exact
    for s in range(S):
        det = OracleTrigger(chunk * 2, 0.8, 1)
        assert [det.update(c) for c in conf[s]] == list(fired[s])
    assert count == fired.sum()
    assert fired.sum() > 0


def test_stream_host_path_equals_device_path():
    m = _mod()
    S, K, chunk = 50, 14, 1024
    pcm = noise(S, K * chunk, seed=9)
    model = m.GruModel.random(13, 20, seed=1, scale=0.1)
    model.dense_b = 3.0
    a = _run_gpu_streams(m, model, pcm, chunk)
    for pinned in (False, True):                    # staged copies / in-place on pinned buffers (n <= 64)
        b = _run_gpu_streams(m, model, pcm, chunk, host=True, pinned=pinned)
        for x, y in zip(a[:4], b[:4]):
            assert np.array_equal(x, y)
        assert a[4] == b[4] and a[4] > 0


def test_host_path_sub_batches_equal_device_path():
    """pb_update_host on 16 400 streams = two pipelined sub-batches (8 224 + 8 176: the first runs the tensor-core scan, the
    second the warp-per-stream kernel) with a weight reload in between: must equal the single-launch device path."""
    m = _mod()
    S, K, chunk = 16400, 32, 1024
    pcm = noise(64, K * chunk, seed=41)
    pcm = np.tile(pcm, (S // 64 + 1, 1))[:S].copy()
    pcm[::5] = np.roll(pcm[::5], 321, axis=1)
    model = m.GruModel.random(13, 20, seed=12, scale=0.1)
    model.dense_b = 3.0
    dev = m.StreamBatch(model, S, chunk_samples=chunk)
    host = m.StreamBatch(model, S, chunk_samples=chunk)
    conf = np.zeros(S); raw = np.zeros(S, np.float32); fired = np.zeros(S, np.uint8)
    total = 0
    for k in range(K):
        c = np.ascontiguousarray(pcm[:, k * chunk:(k + 1) * chunk])
        if k == 27:
            for sb in (dev, host):
                sb.core.load_weights(model.kernel, model.recurrent, model.bias, model.dense_w, model.dense_b)
        o = dev.update(cuda(c))
        total += host.update_host(c, conf, raw, fired)
        assert np.max(np.abs(o['raw'].cpu().numpy() - raw)) < 1e-6, k
        assert np.array_equal(o['fired'].cpu().numpy().astype(bool), fired.astype(bool)), k
    assert total == int(dev.count.item()) > 0
    dev.core.close(); host.core.close()


def test_handles_with_different_geometries_coexist():
    """Kernel attributes (dynamic shared memory limits) are per kernel, not per handle: creating a small-geometry handle
    after a large one must not break the large one's launches."""
    m = _mod()
    chunk = 1024
    pcm = noise(6, 40 * chunk, seed=43)
    pr_big = m.ListenerParams(n_filt=40, n_mfcc=40)
    big_model = m.GruModel.random(40, 128, seed=2, scale=0.1 / np.sqrt(128 / 20.0))
    tiled_model = m.GruModel.random(26, 64, seed=3, scale=0.1 / np.sqrt(64 / 20.0))     # tiled kernel, 56 KB of dynamic smem
    big = m.StreamBatch(big_model, 6, params=pr_big, chunk_samples=chunk)
    tiled = m.StreamBatch(tiled_model, 6, params=m.ListenerParams(use_delta=True), chunk_samples=chunk)
    small = m.StreamBatch(m.GruModel.random(13, 20, seed=4, scale=0.1), 6, chunk_samples=chunk)      # created last
    tiny = m.StreamBatch(m.GruModel.random(26, 8, seed=5, scale=0.1), 6, params=m.ListenerParams(use_delta=True),
                         chunk_samples=chunk)                                                        # tiled kernel again, 13 KB
    outs = {}
    for k in range(40):
        c = cuda(pcm[:, k * chunk:(k + 1) * chunk])
        for name, sb in (('big', big), ('tiled', tiled), ('small', small), ('tiny', tiny)):
            outs.setdefault(name, []).append(sb.update(c)['raw'].cpu().numpy().copy())
    w = og.GruWeights(big_model.kernel, big_model.recurrent, big_model.bias, big_model.dense_w, big_model.dense_b)
    oraw, _, _ = run_streams(w, pcm, chunk, pr=OracleParams(**pr_big.to_dict()))
    assert np.max(np.abs(np.array(outs['big']).T - oraw)) < 1e-4
    w = og.GruWeights(tiled_model.kernel, tiled_model.recurrent, tiled_model.bias, tiled_model.dense_w, tiled_model.dense_b)
    oraw, _, _ = run_streams(w, pcm, chunk, pr=OracleParams(**m.ListenerParams(use_delta=True).to_dict()))
    assert np.max(np.abs(np.array(outs['tiled']).T - oraw)) < 1e-4
    got = big.core.mfcc(cuda(pcm[:, :8000])).cpu().numpy()                 # batch MFCC kernels of the large geometry as well
    assert got.shape[-1] == 40 and np.isfinite(got).all()
    for sb in (big, tiled, small, tiny):
        sb.core.close()


def test_stream_ids_subset_and_clear():
    m = _mod()
    S, chunk = 16, 1024
    model = m.GruModel.random(13, 20, seed=2, scale=0.1)
    pcm = noise(S, 20 * chunk, seed=11)
    sb = m.StreamBatch(model, S, chunk_samples=chunk)
    ids = torch.tensor([3, 9, 4, 15], dtype=torch.int32, device='cuda')
    ref = m.StreamBatch(model, 4, chunk_samples=chunk)
    for k in range(10):
        c = pcm[:, k * chunk:(k + 1) * chunk]
        a = sb.update(cuda(c[[3, 9, 4, 15]]), ids)
        b = ref.update(cuda(c[[3, 9, 4, 15]]))
        assert torch.equal(a['conf'], b['conf']) and torch.equal(a['raw'], b['raw'])
    # untouched streams are still in their initial state
    assert float(sb.core.read_window(S)[0].abs().max()) == 0.0
    # clear two of them: they behave like fresh streams afterwards
    cl = torch.tensor([9, 15], dtype=torch.int32, device='cuda')
    sb.clear(cl)
    fresh = m.StreamBatch(model, 2, chunk_samples=chunk)
    for k in range(10, 16):
        c = pcm[:, k * chunk:(k + 1) * chunk]
        a = sb.update(cuda(c[[9, 15]]), cl)
        b = fresh.update(cuda(c[[9, 15]]))
        assert torch.equal(a['conf'], b['conf'])
    for x in (sb, ref, fresh):
        x.core.close()


def test_stream_config3_and_delta_and_mels():
    m = _mod()
    chunk, S, K = 1024, 5, 40
    pcm = noise(S, K * chunk, seed=13)
    for kw, H in ((dict(n_filt=40, n_mfcc=40), 128), (dict(use_delta=True), 20)):
        pr = m.ListenerParams(**kw)
        F = pr.feature_size
        model = m.GruModel.random(F, H, seed=3, scale=0.1 / np.sqrt(H / 20.0))
        raw, conf, fired, wins, count = _run_gpu_streams(m, model, pcm, chunk, pr=pr)
        w = og.GruWeights(model.kernel, model.recurrent, model.bias, model.dense_w, model.dense_b)
        oraw, oconf, ofired = run_streams(w, pcm, chunk, pr=OracleParams(**pr.to_dict()))
        print(kw, 'raw err', np.max(np.abs(raw - oraw)))
        assert np.max(np.abs(raw - oraw)) < 1e-4


def test_mels_vectorizer():
    m = _mod()
    pr = m.ListenerParams(vectorizer=m.Vectorizer.mels)
    c = m.PreciseB200(pr)
    pcm = noise(3, 8000, seed=17)
    got = c.mfcc(cuda(pcm)).cpu().numpy()
    want = np.stack([om.mel_spec(r.astype(np.float32) / 32768.0, 16000, 1600, 800, 512, 20) for r in pcm])
    assert got.shape == want.shape and np.max(np.abs(got - want)) < 2e-4
    c.close()


@pytest.mark.parametrize('kw', [dict(n_fft=256), dict(n_fft=128, window_t=0.02, hop_t=0.01), dict(n_fft=64, n_filt=12, n_mfcc=8),
                                dict(n_fft=256, window_t=0.01, hop_t=0.005), dict(n_fft=1024), dict(n_fft=1024, window_t=0.05, hop_t=0.02, n_filt=26),
                                dict(n_fft=1024, hop_t=0.005)])
def test_generic_n_fft(kw):
    """n_fft is a ListenerParams field (precise/params.py:49); any power of two in [64, 1024] other than 512 runs through the radix-2
    path (1024: crop to 1024 of 1600 samples, zero-pad of an 800-sample window, and 13+ frames per tick at hop_t = 0.005).
    Covers crop (window > n_fft) and zero-pad (window < n_fft) framing, batch and streaming."""
    m = _mod()
    pr = m.ListenerParams(**kw)
    opr = OracleParams(**pr.to_dict())
    c = m.PreciseB200(pr)
    pcm = noise(5, 9000, seed=23)
    got = c.mfcc(cuda(pcm)).cpu().numpy()
    want = np.stack([om.mfcc_spec(r.astype(np.float32) / 32768.0, 16000, pr.window_samples, pr.hop_samples,
                                  pr.n_fft, pr.n_filt, pr.n_mfcc) for r in pcm])
    assert got.shape == want.shape
    print(kw, 'mfcc err', np.max(np.abs(got - want)))
    assert np.max(np.abs(got - want)) < 2e-4
    c.close()
    chunk = 1024 if pr.n_fft == 1024 else min(1024, 4 * pr.hop_samples)
    pcm = noise(4, 24 * chunk, seed=29)
    model = m.GruModel.random(pr.feature_size, 20, seed=5, scale=0.1)
    raw, conf, fired, wins, count = _run_gpu_streams(m, model, pcm, chunk, pr=pr)
    w = og.GruWeights(model.kernel, model.recurrent, model.bias, model.dense_w, model.dense_b)
    oraw, oconf, ofired = run_streams(w, pcm, chunk, pr=opr)
    assert np.max(np.abs(raw - oraw)) < 1e-4 and np.array_equal(fired, ofired)


@pytest.mark.parametrize('kw,chunk', [(dict(hop_t=0.005), 1024), (dict(), 8000), (dict(), 12345), (dict(hop_t=0.02, window_t=0.05), 3000)],
                         ids=['hop80_chunk1024', 'chunk8000', 'chunk12345_odd', 'hop320_chunk3000'])
def test_many_frames_per_tick(kw, chunk):
    """Chunks that complete more than 8 frames per stream and tick (the reference featurises whatever its carry buffer holds,
    network_runner.py:139-144): fed as sub-chunks through the generic kernel, the network once per tick.  Windows, raw outputs
    and detections against independent oracle Listeners, including the 13-frames-per-tick geometry hop_t = 0.005 / chunk 1024."""
    m = _mod()
    pr = m.ListenerParams(**kw)
    opr = OracleParams(**pr.to_dict())
    S, K = 5, max(6, 40000 // chunk)
    pcm = noise(S, K * chunk, seed=chunk)
    pcm[3] = 0
    model = m.GruModel.random(pr.feature_size, 20, seed=5, scale=0.1)
    raw, conf, fired, wins, count = _run_gpu_streams(m, model, pcm, chunk, pr=pr, sens=0.8, lvl=1)
    owins = _oracle_windows(pcm, chunk, opr)
    assert np.max(np.abs(wins - owins)) < 2e-4
    w = og.GruWeights(model.kernel, model.recurrent, model.bias, model.dense_w, model.dense_b)
    oraw, oconf, ofired = run_streams(w, pcm, chunk, pr=opr, sensitivity=0.8, trigger_level=1)
    assert np.max(np.abs(raw - oraw)) < 1e-4 and np.array_equal(fired, ofired)
    assert count == fired.sum()


@pytest.mark.parametrize('kw', [dict(), dict(n_filt=26, n_mfcc=13), dict(window_t=0.05, hop_t=0.02)], ids=['default', 'filt26', 'window800'])
def test_speechpy_vectorizer(kw):
    """Vectorizer.speechpy_mfccs (legacy .params files, precise/params.py:147; precise/vectorization.py:40-42), PARITY UNPINNED: against the
    oracle's restatement of speechpy's published algorithm (mel corners up to sample_rate / 2 on floor((n_bins + 1) hz / sr), one frame
    fewer than sonopy's framing).  Batch featuriser, then the stateful tick against oracle Listeners (windows, raw, detections)."""
    m = _mod()
    pr = m.ListenerParams(vectorizer=m.Vectorizer.speechpy_mfccs, **kw)
    opr = OracleParams(**pr.to_dict())
    c = m.PreciseB200(pr)
    pcm = noise(5, 9000, seed=41)
    pcm[4] = 0
    got = c.mfcc(cuda(pcm)).cpu().numpy()
    want = np.stack([om.speechpy_mfcc(r.astype(np.float32) / 32768.0, 16000, pr.window_samples, pr.hop_samples, pr.n_fft, pr.n_filt, pr.n_mfcc)
                     for r in pcm])
    assert got.shape == want.shape and got.shape[1] > 0
    assert np.max(np.abs(got - want)) < 2e-4
    c.close()
    chunk = 1024
    pcm = noise(4, 30 * chunk, seed=43)
    model = m.GruModel.random(pr.feature_size, 20, seed=5, scale=0.1)
    raw, conf, fired, wins, count = _run_gpu_streams(m, model, pcm, chunk, pr=pr, sens=0.8, lvl=1)
    owins = _oracle_windows(pcm, chunk, opr)
    assert np.max(np.abs(wins - owins)) < 2e-4
    w = og.GruWeights(model.kernel, model.recurrent, model.bias, model.dense_w, model.dense_b)
    oraw, oconf, ofired = run_streams(w, pcm, chunk, pr=opr, sensitivity=0.8, trigger_level=1)
    assert np.max(np.abs(raw - oraw)) < 1e-4 and np.array_equal(fired, ofired)


def test_gru_mode_accepts_only_existing_kernels(core):
    """pb_debug_gru_mode: 0 (automatic), 1 (CUDA cores) and 2 (tensor cores) select a kernel; any other mode is refused."""
    try:
        for mode in (0, 1, 2):
            core.gru_mode(mode)
        for mode in (-1, 3, 7, 9, 10, 11):
            with pytest.raises(ValueError, match='gru mode'):
                core.gru_mode(mode)
    finally:
        core.gru_mode(0)


def test_unsupported_and_errors():
    m = _mod()
    with pytest.raises(NotImplementedError):
        m.PreciseB200(m.ListenerParams(n_fft=2048))
    with pytest.raises(NotImplementedError):
        m.PreciseB200(m.ListenerParams(n_fft=384))
    c = m.PreciseB200(max_streams=4)
    with pytest.raises(m.PBError):
        c.predict(torch.zeros((1, 29, 13), device='cuda'))           # weights not loaded
    with pytest.raises(ValueError):
        c.update(torch.zeros((5, 1024), dtype=torch.int16, device='cuda'))   # n > max_streams
    c.close()


# ------------------------------------------------------------------------------------------ mirrors
def test_listener_and_engine_mirrors_vs_reference_listener(golden_dir):
    """B200Listener / B200Engine on the PCM of the golden fixture that the reference's real Listener produced."""
    import os
    m = _mod()
    g = np.load(os.path.join(golden_dir, 'listener_golden.npz'))
    model = m.GruModel(g['kernel'], g['recurrent'], g['bias'], g['dense_w'], g['dense_b'])
    d = OracleDecoder(((6, 4),), 0.2)
    step = np.max(np.abs(np.diff(d.cd))) * 2.5
    for i, chunk in ((0, 1024), (3, 3000), (4, 333)):
        pcm = g['pcm_%d' % i]
        want = g['conf_%d' % i]
        lis = m.B200Listener(model, chunk * 2)
        got = np.array([lis.update(pcm[k * chunk:(k + 1) * chunk].tobytes()) for k in range(len(want))])
        # golden weights (scale 0.3) saturate quickly; compare where the oracle is not pinned at 0/1
        assert np.max(np.abs(got - want)) < 5e-3, (i, np.max(np.abs(got - want)))
        with pytest.raises(EOFError):
            lis.update(b'')
    pcm, want = g['pcm_0'], g['conf_0']
    eng = m.B200Engine(model, 2048)
    eng.start()
    got = np.array([eng.get_prediction(pcm[k * 1024:(k + 1) * 1024].tobytes()) for k in range(len(want))])
    with pytest.raises(ValueError):
        eng.get_prediction(b'\0' * 100)
    eng.stop()
    assert np.max(np.abs(got - want)) < 5e-3


def test_listener_mirror_vs_reference_listener_tight(golden_dir):
    """The reference's real Listener (imported in the build container, make_golden.py) with well-conditioned weights (0.1-scaled:
    outputs away from saturation): every confidence of the GPU mirror equals the reference's, except that a float32 network
    output one ulp off may pick the neighbouring LUT bin; measured flip rate printed, bounded at 2 %, never more than one bin."""
    import os
    m = _mod()
    g = np.load(os.path.join(golden_dir, 'listener_golden_s01.npz'))
    model = m.GruModel(g['kernel'], g['recurrent'], g['bias'], g['dense_w'], g['dense_b'])
    d = OracleDecoder(((6, 4),), 0.2)
    step = np.max(np.abs(np.diff(d.cd))) * 1.01 / 0.2 * 0.5          # one LUT bin after the piecewise-linear remap (centre 0.2)
    flips = total = 0
    for i in range(8):
        if 'pcm_%d' % i not in g.files:
            break
        pcm, want, chunk = g['pcm_%d' % i], g['conf_%d' % i], int(g['chunk_%d' % i])
        lis = m.B200Listener(model, chunk * 2)
        got = np.array([lis.update(pcm[k * chunk:(k + 1) * chunk].tobytes()) for k in range(len(want))])
        assert np.max(np.abs(got - want)) <= step, (i, np.max(np.abs(got - want)), step)
        flips += int(np.sum(got != want)); total += len(want)
    print('listener golden (0.1-scaled weights): %d / %d confidences differ by one LUT bin' % (flips, total))
    assert flips <= 0.02 * total


def test_runner_plugin_predict_shape():
    m = _mod()
    model = m.GruModel.random(13, 20, seed=4, scale=0.1)
    r = m.B200Runner(model)
    x = np.random.RandomState(0).randn(9, 29, 13)
    p = r.predict(x)
    assert p.shape == (9, 1) and p.dtype == np.float32
    assert abs(r.run(x[2]) - p[2, 0]) < 1e-7


@pytest.mark.parametrize('k1_mode', [3, 4, 5, 6], ids=['fft_64bit_setup', 'tensor_core', 'tensor_core_two_stage', 'two_stage_shuffle_epilogue'])
def test_alternative_mfcc_tick_kernels(k1_mode):
    """pb_debug_k1_mode against the default kernel (FFT on the CUDA cores, 32-bit per-pass set-up): 3 = the same kernel with its
    original 64-bit set-up (must be bit-identical: same arithmetic, different address computation), 4 = the mma.sync DFT tick
    (mfcc_mma.cuh) with stage 1 on the CUDA cores, 5 = both stages on the tensor cores from exactly split int16 samples,
    6 = 5 with the shuffle epilogue."""
    m = _mod()
    chunk, S, K = 1024, 300, 40
    pcm = noise(S, K * chunk, seed=51)
    pcm[0] = 0; pcm[1] = 32767; pcm[2] = -32768
    model = m.GruModel.random(13, 20, seed=9, scale=0.1)
    ref = m.StreamBatch(model, S, chunk_samples=chunk)
    ref.core.k1_mode(2)                               # the FFT kernel whatever the batch size
    tc = m.StreamBatch(model, S, chunk_samples=chunk)
    tc.core.k1_mode(k1_mode)
    for k in range(K):
        c = cuda(pcm[:, k * chunk:(k + 1) * chunk])
        a, b = ref.update(c), tc.update(c)
        wa, wb = ref.core.read_window(S).cpu().numpy(), tc.core.read_window(S).cpu().numpy()
        per = np.abs(wa - wb).reshape(S, -1).max(1)
        assert np.max(per) < 2e-4, k
        if k1_mode == 3:
            assert np.array_equal(wa, wb), k
        assert np.max(np.abs(a['raw'].cpu().numpy() - b['raw'].cpu().numpy())) < 1e-4, k
    ref.core.close(); tc.core.close()


@pytest.mark.parametrize('chunk', [1024, 800, 2000, 1600])
def test_two_stage_tensor_core_mfcc_vs_oracle_ragged(chunk):
    """k1 mode 5 (mfcc_mma.cuh: plan kernel + both DFT stages on mma.sync) against independent oracle Listeners: windows after every
    tick, with streams of different ages in one batch (id subsets skip ticks), several frames per tick (chunk 1600 / 2000), silent,
    full-scale DC, near-silent and boundary-hovering streams, and a partial last tile (frames not a multiple of 32)."""
    import torch
    m = _mod()
    S, K = 77, max(10, 24000 // chunk)
    pcm = noise(S, K * chunk, seed=chunk + 5)
    pcm[5] = 0
    pcm[6] = 32767
    pcm[7] = -32768
    rs = np.random.RandomState(3)
    pcm[8] = np.round(rs.randn(K * chunk) * 1.5)
    pcm[9] = 128 + np.round(rs.randn(K * chunk) * 2)
    pcm[10] = -20000 + np.round(rs.randn(K * chunk) * 300)
    model = m.GruModel.random(13, 20, seed=0, scale=0.1)
    sb = m.StreamBatch(model, S, chunk_samples=chunk)
    sb.core.k1_mode(5)
    opr = OracleParams()
    w = og.GruWeights(model.kernel, model.recurrent, model.bias, model.dense_w, model.dense_b)
    lis = [OracleListener(w, opr) for _ in range(S)]
    fed = np.zeros(S, int)                         # chunks each stream has consumed
    worst = 0.0
    for k in range(K):
        # even ticks: every stream; odd ticks: a shuffled subset (the others fall behind -> different ages / tails)
        ids = np.arange(S) if k % 2 == 0 else rs.permutation(S)[:S // 2 + k % 5]
        c = np.stack([pcm[i, fed[i] * chunk:(fed[i] + 1) * chunk] for i in ids])
        sb.update(cuda(c), ids=torch.from_numpy(ids.astype(np.int32)).cuda())
        win = sb.core.read_window(S).cpu().numpy()
        for j, i in enumerate(ids):
            ow = lis[i].update_vectors(c[j].astype(np.float32) / 32768.0)
            worst = max(worst, float(np.max(np.abs(win[i] - ow))))
            fed[i] += 1
    print('chunk', chunk, 'max |window - oracle|', worst)
    assert worst < 2e-4
    sb.core.close()


def test_default_kernel_choice_large_tick_matches_fft_kernel():
    """A large tick (49 189 streams: 16 streams per warp tile, several tiles per warp, partial last tile) through the default
    MFCC kernel (FFT, 32-bit per-pass set-up) must give the same windows, network outputs and detections as the FFT kernel
    with its original 64-bit set-up on the same audio: the two differ only in address arithmetic."""
    m = _mod()
    chunk, S, K = 1024, 49152 + 37, 30
    base = noise(256, K * chunk, seed=77)
    base[3] = 0; base[4] = 32767; base[5] = np.round(np.random.RandomState(1).randn(K * chunk) * 2)
    pcm = np.tile(base, (S // 256 + 1, 1))[:S]
    model = m.GruModel.random(13, 20, seed=9, scale=0.1)
    model.dense_b = 3.0
    a = m.StreamBatch(model, S, chunk_samples=chunk, sensitivity=0.9, trigger_level=0)
    b = m.StreamBatch(model, S, chunk_samples=chunk, sensitivity=0.9, trigger_level=0)
    b.core.k1_mode(3)
    worst = 0.0
    for k in range(K):
        c = cuda(np.ascontiguousarray(pcm[:, k * chunk:(k + 1) * chunk]))
        ra, rb = a.update(c), b.update(c)
        worst = max(worst, float((ra['raw'] - rb['raw']).abs().max().item()))
        if k % 7 == 6 or k == K - 1:
            wa, wb = a.core.read_window(S), b.core.read_window(S)
            assert torch.equal(wa, wb), k
    assert worst == 0.0
    ca, cb = int(a.count.item()), int(b.count.item())
    assert ca > 0 and ca == cb, (ca, cb)
    a.core.close(); b.core.close()


def test_two_stage_tensor_core_mfcc_large_tick_matches_fft_kernel():
    """k1 mode 5 (mfcc_mma.cuh) at 20 011 streams per tick (2 500 to 3 200 tiles of 8 frames: several tiles per warp, partial last tile)
    against the FFT kernel on the same audio: windows, network outputs and detections."""
    m = _mod()
    chunk, S, K = 1024, 20011, 30
    base = noise(256, K * chunk, seed=78)
    base[3] = 0; base[4] = 32767; base[5] = np.round(np.random.RandomState(2).randn(K * chunk) * 2)
    pcm = np.tile(base, (S // 256 + 1, 1))[:S]
    model = m.GruModel.random(13, 20, seed=9, scale=0.1)
    model.dense_b = 3.0
    a = m.StreamBatch(model, S, chunk_samples=chunk, sensitivity=0.9, trigger_level=0)
    b = m.StreamBatch(model, S, chunk_samples=chunk, sensitivity=0.9, trigger_level=0)
    a.core.k1_mode(5)
    b.core.k1_mode(2)
    worst = 0.0
    for k in range(K):
        c = cuda(np.ascontiguousarray(pcm[:, k * chunk:(k + 1) * chunk]))
        ra, rb = a.update(c), b.update(c)
        worst = max(worst, float((ra['raw'] - rb['raw']).abs().max().item()))
        if k % 7 == 6 or k == K - 1:
            wa, wb = a.core.read_window(S), b.core.read_window(S)
            assert float((wa - wb).abs().max().item()) < 2e-4, k
    assert worst < 1e-4
    ca, cb = int(a.count.item()), int(b.count.item())
    assert ca > 0 and abs(ca - cb) <= max(3, ca // 5000), (ca, cb)
    a.core.close(); b.core.close()


def test_detection_counter_overlapped_allreduce_single_rank():
    """DetectionCounter.all_reduce_overlapped (snapshot on the compute stream, reduce on a side stream) follows the device counter."""
    import torch
    from mycroft_precise_b200.dist import DetectionCounter
    local = torch.zeros(1, dtype=torch.int64, device='cuda')
    c = DetectionCounter(local)
    for k in range(7):
        local += k + 1
        c.all_reduce_overlapped()
    c.wait()
    torch.cuda.synchronize()
    assert int(c.total.item()) == int(local.item()) == 28

