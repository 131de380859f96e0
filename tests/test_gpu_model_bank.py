"""Model bank: several networks scored per tick over one MFCC front end (pb_add_model / pb_update_models, gru_bank.cuh).

-m gpu, except the C-ABI null-handle check at the end.  Tolerances as in test_gpu_parity.py: raw 1e-5 against the float64
GRU on the GPU's own windows, 1e-4 end to end against the oracle listeners, conf up to a neighbouring LUT bin, trigger exact.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import gru as og
from oracle.decoder import OracleDecoder
from oracle.listener import run_streams
from oracle.params import OracleParams
from oracle.trigger import OracleTrigger

gpu = pytest.mark.gpu


def _mod():
    import mycroft_precise_b200 as m
    return m


def cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def noise(S, L, seed=0, sigma=3000):
    rs = np.random.RandomState(seed)
    return np.clip(rs.randn(S, L) * sigma, -32768, 32767).astype(np.int16)


def weights(model):
    return og.GruWeights(model.kernel, model.recurrent, model.bias, model.dense_w, model.dense_b,
                         model.activation, model.recurrent_activation)


def neighbour_ok(d, r, got):
    """got is the decoder's value for raw r or that of a LUT bin next to it (CUDA log vs libm log)."""
    want = d.decode(r)
    if got == want:
        return True
    i = d.index(r)
    for j in (i - 1, i + 1):
        if 0 <= j < len(d.cd):
            cp = d.cd[j]
            if got == (0.5 * cp / d.center if cp < d.center else 0.5 + 0.5 * (cp - d.center) / (1 - d.center)):
                return True
    return False


def bank_models(m):
    """(model, ListenerParams or None, sensitivity, trigger_level) of the four-model bank: the default network, a small one
    with its own decoder and trigger, tanh / sigmoid activations, and H = 32 (outside the fused family)."""
    m0 = m.GruModel.random(13, 20, seed=0, scale=0.1)
    m1 = m.GruModel.random(13, 12, seed=1, scale=0.1)
    m2 = m.GruModel.random(13, 20, seed=2, scale=0.1)
    m2.activation, m2.recurrent_activation = 'tanh', 'sigmoid'
    m3 = m.GruModel.random(13, 32, seed=3, scale=0.1 / np.sqrt(32 / 20.0))
    p1 = m.ListenerParams(threshold_config=((8, 3),), threshold_center=0.3)
    return [(m0, None, 0.8, 1), (m1, p1, 0.8, 1), (m2, None, 0.5, 3), (m3, None, 0.5, 3)]


@gpu
@pytest.mark.parametrize('chunk', [1024, 333])
def test_bank_vs_oracle(chunk):
    m = _mod()
    S, K = 7, max(12, 30000 // chunk)
    pcm = noise(S, K * chunk, seed=chunk)
    pcm[5] = 0
    pcm[6] = 32767
    spec = bank_models(m)
    sb = m.StreamBatch(spec[0][0], S, chunk_samples=chunk, sensitivity=spec[0][2], trigger_level=spec[0][3])
    for i, (model, pr, sens, lvl) in enumerate(spec[1:], 1):
        assert sb.add_model(model, pr, sensitivity=sens, trigger_level=lvl) == i
    M = len(spec)
    assert sb.core.num_models == M
    raw = np.zeros((M, S, K), np.float32)
    conf = np.zeros((M, S, K))
    fired = np.zeros((M, S, K), bool)
    wins = []
    for k in range(K):
        o = sb.update_models(cuda(pcm[:, k * chunk:(k + 1) * chunk]))
        assert tuple(o['conf'].shape) == (M, S)
        raw[:, :, k] = o['raw'].cpu().numpy()
        conf[:, :, k] = o['conf'].cpu().numpy()
        fired[:, :, k] = o['fired'].cpu().numpy().astype(bool)
        wins.append(sb.core.read_window(S).cpu().numpy())
    wins = np.array(wins).reshape(-1, 29, 13)
    counts = sb.counts.cpu().numpy()
    for i, (model, pr, sens, lvl) in enumerate(spec):
        w = weights(model)
        opr = OracleParams(**(pr or m.ListenerParams()).to_dict())
        p64 = og.gru_forward(w, wins, np.float64)[0].reshape(K, S).T
        err64 = np.max(np.abs(raw[i] - p64))
        oraw, _, _ = run_streams(w, pcm, chunk, pr=opr, sensitivity=sens, trigger_level=lvl)
        err = np.max(np.abs(raw[i] - oraw))
        print('model %d (H=%d %s/%s): |raw - f64 GRU on GPU windows| %.3g, |raw - oracle| %.3g, fired %d'
              % (i, model.hidden, model.activation, model.recurrent_activation, err64, err, fired[i].sum()))
        assert err64 < 1e-5 and err < 1e-4
        d = OracleDecoder(opr.threshold_config, opr.threshold_center)
        assert all(neighbour_ok(d, np.float32(r), c) for r, c in zip(raw[i].ravel(), conf[i].ravel()))
        for s in range(S):
            det = OracleTrigger(chunk * 2, sens, lvl)
            assert [det.update(c) for c in conf[i, s]] == list(fired[i, s])
        assert counts[i] == fired[i].sum()
    assert fired.sum() > 0
    sb.core.close()


@gpu
def test_bank_vs_independent_handles_large():
    """9 000 streams (above the warp-per-stream limit), 36 ticks: each bank model against a one-model StreamBatch."""
    m = _mod()
    S, K, chunk = 9000, 36, 1024
    pcm = noise(64, K * chunk, seed=33)
    pcm = np.tile(pcm, (S // 64 + 1, 1))[:S].copy()
    pcm[::7] = np.roll(pcm[::7], 123, axis=1)
    spec = bank_models(m)[:3]
    for model, pr, _, _ in spec:                                     # pushes confidences over the trigger threshold
        model.dense_b = pr.threshold_config[0][0] if pr is not None else 3.0
    bank = m.StreamBatch(spec[0][0], S, chunk_samples=chunk)
    for model, pr, sens, lvl in spec[1:]:
        bank.add_model(model, pr, sensitivity=sens, trigger_level=lvl)
    solo = [m.StreamBatch(model, S, params=pr, chunk_samples=chunk, sensitivity=sens, trigger_level=lvl)
            for model, pr, sens, lvl in spec]
    err = np.zeros(len(spec))
    for k in range(K):
        c = cuda(pcm[:, k * chunk:(k + 1) * chunk])
        o = bank.update_models(c)['raw'].cpu().numpy()
        for i, sb in enumerate(solo):
            err[i] = max(err[i], np.max(np.abs(o[i] - sb.update(c)['raw'].cpu().numpy())))
    counts = bank.counts.cpu().numpy()
    solo_counts = [int(sb.count.item()) for sb in solo]
    print('max |raw bank - one-model handle| per model', err, 'counts', counts, solo_counts)
    assert np.all(err < 1e-5)
    assert all(abs(int(a) - b) <= 3 for a, b in zip(counts, solo_counts)) and counts.min() > 0
    for x in [bank] + solo:
        x.core.close()


@gpu
def test_bank_mixed_with_single_model_api():
    """update (tensor-core scan, > 8192 streams) and update_models alternate on one handle, with a slot-0 weight reload,
    a clear of some streams, an ids-permuted tick and a one-stream tick; independent handles driven through the same
    sequence give the same results (the second model's handle only advances its MFCC state on update ticks)."""
    import torch
    m = _mod()
    S, chunk = 8448, 1024
    pcm = noise(64, 24 * chunk, seed=51)
    pcm = np.tile(pcm, (S // 64 + 1, 1))[:S].copy()
    pcm[::5] = np.roll(pcm[::5], 77, axis=1)
    m0 = m.GruModel.random(13, 20, seed=4, scale=0.1)
    m0.dense_b = 4.0
    m0b = m.GruModel.random(13, 20, seed=5, scale=0.1)
    m0b.dense_b = 4.0
    m1 = m.GruModel.random(13, 12, seed=6, scale=0.1)
    m1.dense_b = 2.0
    bank = m.StreamBatch(m0, S, chunk_samples=chunk)
    bank.add_model(m1, sensitivity=0.7, trigger_level=2)
    a = m.StreamBatch(m0, S, chunk_samples=chunk)
    b = m.StreamBatch(m1, S, chunk_samples=chunk, sensitivity=0.7, trigger_level=2)
    rs = np.random.RandomState(7)
    cleared = torch.from_numpy(np.sort(rs.choice(S, 700, replace=False)).astype(np.int32)).cuda()
    perm = torch.from_numpy(rs.permutation(S).astype(np.int32)).cuda()
    one = torch.tensor([1234], dtype=torch.int32, device='cuda')
    plan = ['bank'] * 6 + ['single'] * 3 + ['bank', 'single', 'reload', 'single', 'clear', 'perm', 'one'] + ['bank'] * 3 + ['single', 'bank']
    fired_bank = np.zeros(2, np.int64)
    fired_solo = np.zeros(2, np.int64)
    err = 0.0
    for k, what in enumerate(plan):
        c = pcm[:, k * chunk:(k + 1) * chunk]
        if what == 'reload':
            for x in (bank, a):
                x.core.load_weights(m0b.kernel, m0b.recurrent, m0b.bias, m0b.dense_w, m0b.dense_b)
            what = 'bank'
        if what == 'clear':
            for x in (bank, a, b):
                x.clear(cleared)
            what = 'bank'
        ids, cc = None, c
        if what == 'perm':
            ids, cc = perm, c[perm.cpu().numpy()]
        elif what == 'one':
            ids, cc = one, c[1234:1235]
        if what == 'single':
            o = bank.update(cuda(cc), ids)['raw'].cpu().numpy()
            err = max(err, np.max(np.abs(o - a.update(cuda(cc), ids)['raw'].cpu().numpy())))
            b.core.update_vectors(cuda(cc), ids)
            continue
        o = bank.update_models(cuda(cc), ids)
        raw, fired = o['raw'].cpu().numpy(), o['fired'].cpu().numpy()
        fired_bank += fired.sum(axis=1).astype(np.int64)
        for i, x in enumerate((a, b)):
            ox = x.update(cuda(cc), ids)
            err = max(err, np.max(np.abs(raw[i] - ox['raw'].cpu().numpy())))
            fired_solo[i] += int(ox['fired'].sum())
    print('max |raw| difference %.3g; fired on bank ticks: bank %s, independent handles %s' % (err, fired_bank, fired_solo))
    assert err < 1e-5
    assert np.array_equal(bank.counts.cpu().numpy(), fired_bank)
    assert np.all(np.abs(fired_bank - fired_solo) <= 3) and fired_bank.min() > 0
    for x in (bank, a, b):
        x.core.close()


@gpu
def test_bank_errors(tmp_path):
    import torch
    m = _mod()
    from mycroft_precise_b200.core import PBError
    from mycroft_precise_b200.params import save_params
    sb = m.StreamBatch(m.GruModel.random(13, 20, seed=0, scale=0.1), 16)
    with pytest.raises(ValueError, match='n_mfcc'):
        sb.add_model(m.GruModel.random(12, 20, seed=1), m.ListenerParams(n_mfcc=12))
    with pytest.raises(ValueError, match='features'):
        sb.add_model(m.GruModel.random(12, 20, seed=1))
    path = str(tmp_path / 'other.npz')                      # a weights file whose .params file has another front end
    m.save_weights(path, m.GruModel.random(13, 20, seed=2))
    save_params(path, m.ListenerParams(hop_t=0.04))
    with pytest.raises(ValueError, match='hop_samples'):
        sb.add_model(path)
    save_params(path, m.ListenerParams(threshold_center=0.4))
    assert sb.add_model(path) == 1                           # same front end, its own decoder
    for i in range(2, 8):
        assert sb.add_model(m.GruModel.random(13, 8 + i, seed=10 + i, scale=0.1)) == i
    with pytest.raises(ValueError, match='at most 8'):
        sb.add_model(m.GruModel.random(13, 20, seed=20))
    assert sb.core.num_models == 8 and tuple(sb.counts.shape) == (8,)
    o = sb.update_models(torch.zeros((16, 1024), dtype=torch.int16, device='cuda'))
    assert tuple(o['raw'].shape) == (8, 16)
    sb.reset_count()
    assert int(sb.counts.abs().sum()) == 0
    c = m.PreciseB200(max_streams=4)
    with pytest.raises(PBError):
        c.update_models(torch.zeros((4, 1024), dtype=torch.int16, device='cuda'))
    with pytest.raises(ValueError):
        c.update_models(torch.zeros((4, 1024), dtype=torch.int16, device='cuda'), counts=torch.zeros(2, dtype=torch.int64, device='cuda'))
    for x in (sb.core, c):
        x.close()


def test_add_model_null_handle_is_invalid():
    import os
    import __graft_entry__ as g
    from mycroft_precise_b200.core import lib_path, get_lib, pb_config
    if not os.path.isfile(lib_path()):
        g.build()
    lib = get_lib()
    cfg = pb_config()
    assert lib.pb_config_default(C.byref(cfg)) == 0
    w = np.zeros(3 * 20 * 33, np.float32)
    p = w.ctypes.data_as(C.c_void_p)
    slot = C.c_int32(-7)
    assert lib.pb_add_model(None, C.byref(cfg), p, p, p, p, 0.0, None, 0, C.byref(slot)) == -1
    assert b'null' in lib.pb_last_error() and slot.value == -7
    assert lib.pb_num_models(None) == -1
    assert lib.pb_update_models(None, None, None, 0, None, None, None, None, None) == -1
