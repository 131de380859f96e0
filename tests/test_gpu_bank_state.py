"""Model-bank state across a failed pb_add_model and across pb_clear (-m gpu).

The bank holds two networks gru_bank_kernel scores together (H = 20 and H = 12) and one it scores with its own kernel (H = 32),
each with its own trigger settings.
"""
import ctypes as C

import numpy as np
import pytest

from oracle.trigger import OracleTrigger

gpu = pytest.mark.gpu


def _mod():
    import mycroft_precise_b200 as m
    return m


def cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def pcm_with_pauses(S, K, chunk, seed):
    """Noise that is loud for three chunks, then nearly silent for three, with a different phase per stream."""
    rs = np.random.RandomState(seed)
    t = np.arange(K * chunk) // chunk
    env = np.where(((t[None, :] + np.arange(S)[:, None]) // 3) % 2 == 0, 1.0, 0.05)
    return np.clip(rs.randn(S, K * chunk) * 3000 * env, -32768, 32767).astype(np.int16)


def bank_spec(m):
    """(model, sensitivity, trigger_level); the dense biases push every model's confidences over its threshold."""
    m0 = m.GruModel.random(13, 20, seed=4, scale=0.1)
    m0.dense_b = 3.0
    m1 = m.GruModel.random(13, 12, seed=6, scale=0.1)
    m1.dense_b = 2.0
    m2 = m.GruModel.random(13, 32, seed=8, scale=0.1 / np.sqrt(32 / 20.0))
    m2.dense_b = 3.0
    return [(m0, 0.8, 1), (m1, 0.6, 2), (m2, 0.5, 3)]


def make_bank(m, spec, S, chunk):
    sb = m.StreamBatch(spec[0][0], S, chunk_samples=chunk, sensitivity=spec[0][1], trigger_level=spec[0][2])
    for model, sens, lvl in spec[1:]:
        sb.add_model(model, sensitivity=sens, trigger_level=lvl)
    return sb


def tick(sb, pcm_k):
    o = sb.update_models(cuda(pcm_k))
    return {k: v.cpu().numpy() for k, v in o.items()}


@gpu
def test_failed_add_model_leaves_bank_untouched():
    """A pb_add_model that fails (wrong decoder-table length; a network too large for the tiled kernel) leaves the bank as it
    was: same number of models, and update_models outputs bit-identical to a handle that never saw the failed calls."""
    m = _mod()
    from mycroft_precise_b200.core import make_config, numpy_cdf
    S, K, chunk = 40, 10, 1024
    pcm = pcm_with_pauses(S, K, chunk, seed=71)
    spec = bank_spec(m)
    a, b = make_bank(m, spec, S, chunk), make_bank(m, spec, S, chunk)
    M = len(spec)
    for k in range(K):
        if k == 4:
            core = a.core
            extra = m.GruModel.random(13, 16, seed=9, scale=0.1)
            cfg = make_config(core.params, extra.hidden, core.max_streams, core.chunk_samples, core.device.index)
            kk, u, bb, w = core._weights(core.feature_size, extra.hidden, extra.kernel, extra.recurrent, extra.bias, extra.dense_w)
            cd, _, _ = numpy_cdf(core.params.threshold_config)
            vp = lambda x: x.ctypes.data_as(C.c_void_p)
            slot = C.c_int32(-7)
            rc = core.lib.pb_add_model(core._h, C.byref(cfg), vp(kk), vp(u), vp(bb), vp(w), 0.5, vp(cd), len(cd) - 1, C.byref(slot))
            assert rc == -1 and b'cdf length' in core.lib.pb_last_error() and slot.value == -7
            with pytest.raises(NotImplementedError, match='too large for the tiled GRU kernel'):
                a.add_model(m.GruModel.random(13, 263, seed=10, scale=0.01))
            assert core.num_models == M and b.core.num_models == M
        oa, ob = tick(a, pcm[:, k * chunk:(k + 1) * chunk]), tick(b, pcm[:, k * chunk:(k + 1) * chunk])
        for key in ('raw', 'conf', 'fired'):
            assert oa[key].shape[0] == M
            assert np.array_equal(oa[key], ob[key]), (k, key)
    assert np.array_equal(a.counts.cpu().numpy(), b.counts.cpu().numpy())
    for x in (a, b):
        x.core.close()


@gpu
def test_clear_rearms_every_bank_model():
    """pb_clear of some streams re-arms each model's TriggerDetector on those streams.  Reference: the oracle detector replayed
    on the bank's own confidences, model by model and stream by stream, started afresh where the clear happened."""
    import torch
    m = _mod()
    S, K, chunk, kc = 24, 26, 1024, 14
    pcm = pcm_with_pauses(S, K, chunk, seed=61)
    spec = bank_spec(m)
    sb = make_bank(m, spec, S, chunk)
    M = len(spec)
    cleared = [1, 2, 5, 8, 13, 21]
    conf = np.zeros((M, S, K))
    fired = np.zeros((M, S, K), bool)
    for k in range(K):
        if k == kc:
            sb.clear(torch.tensor(cleared, dtype=torch.int32, device='cuda'))
        o = tick(sb, pcm[:, k * chunk:(k + 1) * chunk])
        conf[:, :, k] = o['conf']
        fired[:, :, k] = o['fired'].astype(bool)
    for i, (model, sens, lvl) in enumerate(spec):
        assert fired[i][cleared, :kc].any(), 'model %d never fired on a cleared stream before the clear' % i
        want = np.zeros((S, K), bool)
        stale = np.zeros((S, K), bool)                        # the same replay without the reset
        for s in range(S):
            det, keep = OracleTrigger(chunk * 2, sens, lvl), OracleTrigger(chunk * 2, sens, lvl)
            for k in range(K):
                if k == kc and s in cleared:
                    det = OracleTrigger(chunk * 2, sens, lvl)
                want[s, k] = det.update(conf[i, s, k])
                stale[s, k] = keep.update(conf[i, s, k])
        print('model %d (H=%d): fired %d, without the re-arm %d' % (i, model.hidden, fired[i].sum(), stale.sum()))
        assert np.array_equal(fired[i], want)
        assert not np.array_equal(fired[i], stale)
    assert np.array_equal(sb.counts.cpu().numpy(), fired.sum(axis=(1, 2)))
    sb.core.close()
