"""Ragged ticks: every stream brings its own number of samples per tick (pb_update_ragged, csrc/mfcc_ragged.cuh).

-m gpu, except the C-ABI null-handle check at the end.  Tolerances as in test_gpu_parity.py: windows 2e-4 against the oracle,
raw 1e-5 against the float64 GRU on the GPU's own windows, raw 1e-4 end to end, conf up to a neighbouring LUT bin, trigger and
counts exact.  Where a ragged tick computes the same thing as a uniform one, the results must be bit-identical.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import gru as og
from oracle.decoder import OracleDecoder
from oracle.listener import OracleListener
from oracle.params import OracleParams
from oracle.trigger import OracleTrigger

gpu = pytest.mark.gpu
LENS = [1, 7, 333, 511, 512, 800, 1024, 4097, 12345]      # 4097 and 12 345 take several MFCC rounds


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
    if got == d.decode(r):
        return True
    i = d.index(r)
    for j in (i - 1, i + 1):
        if 0 <= j < len(d.cd):
            cp = d.cd[j]
            if got == (0.5 * cp / d.center if cp < d.center else 0.5 + 0.5 * (cp - d.center) / (1 - d.center)):
                return True
    return False


def pack(chunks, lead=0):
    """The chunks back to back in one 1-D int16 tensor after `lead` filler samples (odd lead: odd offsets); offsets [n + 1]."""
    offs = lead + np.concatenate([[0], np.cumsum([len(c) for c in chunks])]).astype(np.int64)
    pcm = np.concatenate([np.full(lead, 12345, np.int16)] + [np.asarray(c, np.int16) for c in chunks])
    return cuda(pcm), cuda(offs)


def length_plan(S, K, seed):
    """[K, S] chunk lengths: every length of LENS in the first ticks of every stream, then seeded draws from LENS."""
    rs = np.random.RandomState(seed)
    lens = rs.choice(LENS, size=(K, S))
    for k in range(min(K, len(LENS))):
        lens[k] = [LENS[(k + s) % len(LENS)] for s in range(S)]
    return lens


def streams_audio(S, n, seed):
    audio = [noise(1, n, seed=seed + s)[0] for s in range(S)]
    audio[-2][:] = 0                                      # all-zero stream
    audio[-1][:] = 32767                                  # full-scale DC stream
    return audio


def check_against_oracle(sb, model_i, w, opr, lis, det, chunks, o, S):
    """One tick's outputs of bank model model_i against the stream's oracle Listener (fed the same chunks) and TriggerDetector."""
    raw = o['raw'][model_i].cpu().numpy()
    conf = o['conf'][model_i].cpu().numpy()
    fired = o['fired'][model_i].cpu().numpy().astype(bool)
    win = sb.core.read_window(S).cpu().numpy()
    oraw = np.array([lis[s].update_raw(chunks[s].astype(np.float32) / 32768.0) for s in range(S)], np.float32)
    werr = max(float(np.max(np.abs(win[s] - lis[s].mfccs))) for s in range(S))
    p64 = og.gru_forward(w, win, np.float64)[0].reshape(S)
    d = OracleDecoder(opr.threshold_config, opr.threshold_center)
    assert werr < 2e-4, werr
    assert np.max(np.abs(raw - p64)) < 1e-5 and np.max(np.abs(raw - oraw)) < 1e-4
    assert all(neighbour_ok(d, np.float32(r), c) for r, c in zip(raw, conf))
    assert [det[s].update(conf[s]) for s in range(S)] == list(fired)
    return int(fired.sum())


@gpu
@pytest.mark.parametrize('mode', ['default', 'force_generic', 'n_fft256'])
def test_ragged_vs_oracle(mode):
    """7 streams (one all-zero, one full-scale DC), lengths from LENS, odd and even offsets, against oracle Listeners."""
    m = _mod()
    pr = m.ListenerParams(n_fft=256) if mode == 'n_fft256' else m.ListenerParams()
    opr = OracleParams(**pr.to_dict())
    S, K = 7, 14
    lens = length_plan(S, K, seed=3)
    audio = streams_audio(S, int(lens.sum(axis=0).max()), seed=100)
    model = m.GruModel.random(pr.feature_size, 20, seed=5, scale=0.1)
    sb = m.StreamBatch(model, S, params=pr, sensitivity=0.8, trigger_level=1)
    sb.core.check_ids = True
    if mode == 'force_generic':
        sb.core.force_generic(True)
    w = weights(model)
    lis = [OracleListener(w, opr) for _ in range(S)]
    det = [OracleTrigger(1024 * 2, 0.8, 1) for _ in range(S)]
    pos = np.zeros(S, np.int64)
    fired = 0
    for k in range(K):
        chunks = [audio[s][pos[s]:pos[s] + lens[k, s]] for s in range(S)]
        pos += lens[k]
        pcm, offs = pack(chunks, lead=k % 2)
        o = sb.update_ragged(pcm, offs)
        assert tuple(o['conf'].shape) == (1, S)
        fired += check_against_oracle(sb, 0, w, opr, lis, det, chunks, o, S)
    assert int(sb.counts[0]) == fired
    sb.core.close()


def _uniform_pair(m, S, chunk=1024, model=None):
    model = model or m.GruModel.random(13, 20, seed=7, scale=0.1)
    model.dense_b = 3.0                                  # some streams fire
    return model, m.StreamBatch(model, S, chunk_samples=chunk), m.StreamBatch(model, S, chunk_samples=chunk)


@gpu
@pytest.mark.parametrize('S', [7, 9000])
def test_uniform_ragged_equals_update(S):
    """Every length = chunk_samples, aligned offsets, fresh handle: raw, conf, fired, count and windows equal pb_update's bit for
    bit (7 streams: warp-per-stream network kernel; 9 000: the bank kernel)."""
    import torch
    m = _mod()
    K = 12
    pcm = noise(min(S, 64), K * 1024, seed=11)
    pcm = np.tile(pcm, (S // pcm.shape[0] + 1, 1))[:S].copy()
    pcm[::3] = np.roll(pcm[::3], 77, axis=1)
    _, a, b = _uniform_pair(m, S)
    offs = torch.arange(S + 1, dtype=torch.int64, device='cuda') * 1024
    for k in range(K):
        c = cuda(pcm[:, k * 1024:(k + 1) * 1024])
        oa = a.update(c)
        ob = b.update_ragged(c.view(-1), offs, max_len=1024)
        for key in ('raw', 'conf', 'fired'):
            assert torch.equal(oa[key], ob[key][0]), (k, key)
        assert torch.equal(a.core.read_window(S), b.core.read_window(S))
    assert int(a.count) == int(b.counts[0]) and int(a.count) > 0
    for x in (a, b):
        x.core.close()


@gpu
def test_chunking_independence():
    """Stream 0 gets the audio in 1024-sample chunks, stream 1 the same audio in random splits (ids select who takes part in a
    tick).  Whenever both have consumed the same number of samples, their windows and raw outputs agree to rounding: a row is
    a function of its 512 samples and of the half-warp that computes it (the mel stage's bank-conflict rotation, as in the
    fast kernel), which depends on the frame's place in the tick's frame list.  A staging or state-machine error would move
    a row by orders of magnitude more."""
    import torch
    m = _mod()
    rs = np.random.RandomState(21)
    blocks = [int(q) for q in rs.randint(1, 6, size=10)]          # block j: q_j * 1024 samples
    audio = noise(1, 1024 * sum(blocks), seed=22)[0]
    model = m.GruModel.random(13, 20, seed=8, scale=0.1)
    sb = m.StreamBatch(model, 2)
    pos = 0
    checked = 0
    for q in blocks:
        cuts = np.sort(rs.choice(np.arange(1, q * 1024), size=rs.randint(0, 7), replace=False))
        pieces = np.split(audio[pos:pos + q * 1024], cuts)
        a_pieces = np.split(audio[pos:pos + q * 1024], q)
        last = {}
        for j in range(max(len(pieces), q)):
            items = [(0, a_pieces[j])] if j < q else []
            items += [(1, pieces[j])] if j < len(pieces) else []
            pcm, offs = pack([c for _, c in items], lead=j % 2)
            ids = torch.tensor([i for i, _ in items], dtype=torch.int32, device='cuda')
            o = sb.update_ragged(pcm, offs, ids=ids)['raw'][0]
            for t, (i, _) in enumerate(items):
                last[i] = o[t].item()
        pos += q * 1024
        win = sb.core.read_window(2)
        assert float((win[0] - win[1]).abs().max()) < 1e-5 and abs(last[0] - last[1]) < 1e-6, pos
        checked += 1
    assert checked == len(blocks)
    sb.core.close()


def bank_models(m):
    """The four-model bank of test_gpu_model_bank.py: the default network, a small one with its own decoder and trigger,
    tanh / sigmoid activations, and H = 32 (outside the fused family)."""
    m0 = m.GruModel.random(13, 20, seed=0, scale=0.1)
    m1 = m.GruModel.random(13, 12, seed=1, scale=0.1)
    m2 = m.GruModel.random(13, 20, seed=2, scale=0.1)
    m2.activation, m2.recurrent_activation = 'tanh', 'sigmoid'
    m3 = m.GruModel.random(13, 32, seed=3, scale=0.1 / np.sqrt(32 / 20.0))
    p1 = m.ListenerParams(threshold_config=((8, 3),), threshold_center=0.3)
    return [(m0, None, 0.8, 1), (m1, p1, 0.8, 1), (m2, None, 0.5, 3), (m3, None, 0.5, 3)]


def _bank(m, S, spec):
    sb = m.StreamBatch(spec[0][0], S, sensitivity=spec[0][2], trigger_level=spec[0][3])
    for model, pr, sens, lvl in spec[1:]:
        sb.add_model(model, pr, sensitivity=sens, trigger_level=lvl)
    return sb


@gpu
def test_ragged_model_bank():
    """Four-model bank: ragged ticks checked per model against that model's oracle Listeners; uniform ragged ticks on a fresh
    bank equal update_models bit for bit."""
    import torch
    m = _mod()
    spec = bank_models(m)
    S, K = 7, 11
    lens = length_plan(S, K, seed=4)
    audio = streams_audio(S, int(lens.sum(axis=0).max()), seed=200)
    sb = _bank(m, S, spec)
    M = len(spec)
    opr = [OracleParams(**(pr or m.ListenerParams()).to_dict()) for _, pr, _, _ in spec]
    ws = [weights(model) for model, _, _, _ in spec]
    lis = [[OracleListener(ws[i], opr[i]) for _ in range(S)] for i in range(M)]
    det = [[OracleTrigger(2048, sens, lvl) for _ in range(S)] for _, _, sens, lvl in spec]
    pos = np.zeros(S, np.int64)
    fired = np.zeros(M, np.int64)
    for k in range(K):
        chunks = [audio[s][pos[s]:pos[s] + lens[k, s]] for s in range(S)]
        pos += lens[k]
        pcm, offs = pack(chunks, lead=1 - k % 2)
        o = sb.update_ragged(pcm, offs)
        assert tuple(o['raw'].shape) == (M, S)
        for i in range(M):
            fired[i] += check_against_oracle(sb, i, ws[i], opr[i], lis[i], det[i], chunks, o, S)
    assert np.array_equal(sb.counts.cpu().numpy(), fired)
    sb.core.close()
    a, b = _bank(m, S, spec), _bank(m, S, spec)
    pcm = noise(S, 10 * 1024, seed=5)
    offs = torch.arange(S + 1, dtype=torch.int64, device='cuda') * 1024
    for k in range(10):
        c = cuda(pcm[:, k * 1024:(k + 1) * 1024])
        oa, ob = a.update_models(c), b.update_ragged(c.view(-1), offs)
        for key in ('raw', 'conf', 'fired'):
            assert torch.equal(oa[key], ob[key]), (k, key)
    assert torch.equal(a.counts, b.counts)
    for x in (a, b):
        x.core.close()


@gpu
def test_ragged_mixed_with_uniform_ticks():
    """Ragged ticks with odd lengths leave sample counts that are not multiples of 8; the uniform ticks that follow (update,
    update_models, update_host, update_vectors, a clear, permuted ids) must still match the oracle Listeners.  k1 modes are
    refused on such a handle, and a ragged tick is refused while a k1 mode is set."""
    import torch
    m = _mod()
    from mycroft_precise_b200.core import PBError
    S = 7
    model = m.GruModel.random(13, 20, seed=9, scale=0.1)
    sb = m.StreamBatch(model, S)
    w = weights(model)
    opr = OracleParams()
    lis = [OracleListener(w, opr) for _ in range(S)]
    audio = streams_audio(S, 200000, seed=300)
    pos = np.zeros(S, np.int64)
    rs = np.random.RandomState(31)

    def take(s, L):
        c = audio[s][pos[s]:pos[s] + L]
        pos[s] += L
        return c

    def check(raw, chunks, ids=None):
        """Feed the oracle and compare windows and (if given) raw outputs; raw[i] belongs to stream ids[i]."""
        ids = list(range(S)) if ids is None else list(ids)
        oraw = [lis[s].update_raw(c.astype(np.float32) / 32768.0) for s, c in zip(ids, chunks)]
        win = sb.core.read_window(S).cpu().numpy()
        assert max(float(np.max(np.abs(win[s] - lis[s].mfccs))) for s in range(S)) < 2e-4
        if raw is not None:
            assert np.max(np.abs(np.asarray(raw) - np.asarray(oraw, np.float32))) < 1e-4

    def ragged():
        chunks = [take(s, int(rs.choice([1, 7, 333, 511, 801, 1023, 1501]))) for s in range(S)]
        pcm, offs = pack(chunks, lead=1)
        check(sb.update_ragged(pcm, offs)['raw'][0].cpu().numpy(), chunks)

    def uniform():
        return [take(s, 1024) for s in range(S)]

    ragged()
    with pytest.raises(PBError):
        sb.core.k1_mode(2)
    ragged()
    c = uniform()
    check(sb.update(cuda(np.stack(c)))['raw'].cpu().numpy(), c)
    c = uniform()
    check(sb.update_models(cuda(np.stack(c)))['raw'][0].cpu().numpy(), c)
    c = uniform()
    conf, raw = np.zeros(S), np.zeros(S, np.float32)
    sb.update_host(np.stack(c), conf, raw)
    check(raw, c)
    c = uniform()
    sb.core.update_vectors(cuda(np.stack(c)))
    check(None, c)
    cleared = [1, 4]
    sb.clear(torch.tensor(cleared, dtype=torch.int32, device='cuda'))
    for s in cleared:
        lis[s].clear()
    ragged()
    perm = rs.permutation(S).astype(np.int32)
    c = uniform()
    rows = [c[s] for s in perm]
    check(sb.update(cuda(np.stack(rows)), cuda(perm))['raw'].cpu().numpy(), rows, ids=perm)
    ragged()
    ragged()
    c = uniform()
    check(sb.update(cuda(np.stack(c)))['raw'].cpu().numpy(), c)
    sb.core.close()
    fresh = m.StreamBatch(model, S)
    fresh.core.k1_mode(2)
    with pytest.raises(PBError):
        fresh.update_ragged(torch.zeros(S, dtype=torch.int16, device='cuda'), torch.arange(S + 1, dtype=torch.int64, device='cuda'))
    fresh.core.close()


@gpu
def test_ragged_errors():
    import torch
    m = _mod()
    sb = m.StreamBatch(m.GruModel.random(13, 20, seed=0, scale=0.1), 8)
    sb.core.check_ids = True
    pcm = torch.zeros(4000, dtype=torch.int16, device='cuda')
    t = lambda v: torch.tensor(v, dtype=torch.int64, device='cuda')
    with pytest.raises(ValueError, match='non-decreasing'):
        sb.update_ragged(pcm, t([0, 100, 50, 200]))
    with pytest.raises(ValueError):
        sb.update_ragged(pcm, t([0, 100, 100, 200]))                      # a zero length
    with pytest.raises(ValueError):
        sb.update_ragged(pcm, t([0, 100, 1100, 1200]), max_len=999)       # a length above max_len
    with pytest.raises(ValueError):
        sb.update_ragged(pcm, t([0, 100, 4001]))                          # past the end of pcm
    with pytest.raises(ValueError):
        sb.update_ragged(pcm.view(2, -1), t([0, 100]))
    with pytest.raises(ValueError):
        sb.update_ragged(pcm, t(list(range(10))))                         # 9 streams > max_streams
    o = sb.update_ragged(pcm, t([0, 100, 1100, 1200]), max_len=1000)
    assert tuple(o['conf'].shape) == (1, 3)
    lib, h = sb.core.lib, sb.core._h
    conf = torch.zeros(8, dtype=torch.float64, device='cuda')
    p = C.c_void_p(pcm.data_ptr())
    offs = t([0, 10, 20])
    assert lib.pb_update_ragged(h, p, None, 10, None, 2, None, C.c_void_p(conf.data_ptr()), None, None, None) == -1
    assert lib.pb_update_ragged(h, p, C.c_void_p(offs.data_ptr()), 0, None, 2, None, C.c_void_p(conf.data_ptr()), None, None, None) == -1
    assert lib.pb_update_ragged(h, p, C.c_void_p(offs.data_ptr()), 10, None, 2, None, None, None, None, None) == -1
    assert lib.pb_update_ragged(h, p, C.c_void_p(offs.data_ptr()), 10, None, 9, None, C.c_void_p(conf.data_ptr()), None, None, None) == -1
    torch.cuda.synchronize()
    sb.core.close()
    c = m.PreciseB200(max_streams=4)                                      # no weights: PB_ERR_STATE
    assert c.lib.pb_update_ragged(c._h, p, C.c_void_p(offs.data_ptr()), 10, None, 2, None, C.c_void_p(conf.data_ptr()),
                                  None, None, None) == -4
    c.close()


def test_update_ragged_null_handle_is_invalid():
    import os
    import __graft_entry__ as g
    from mycroft_precise_b200.core import lib_path, get_lib
    if not os.path.isfile(lib_path()):
        g.build()
    lib = get_lib()
    offs = np.zeros(2, np.int64)
    assert lib.pb_update_ragged(None, None, offs.ctypes.data_as(C.c_void_p), 1, None, 1, None, None, None, None, None) == -1
    assert b'null' in lib.pb_last_error()
