"""Stream state export / import (pb_export_streams, pb_import_streams): continuation, round trips, geometries, the ragged rule,
the bank with masks and trigger settings, and validation.

-m gpu, except the C-ABI null-handle check at the end.  A record holds K1's own bits, and a mel-stage row can move by an ulp
with a frame's position in the tick's frame list, so every continuation ticks the source and the destination with the same
items in the same order and maps only the ids: then raw, conf, fired and counts must be equal bit for bit.
"""
import ctypes as C

import numpy as np
import pytest

from test_gpu_model_bank import bank_models
from test_gpu_stream_models import bank, cuda, host, noise
from test_gpu_stream_trigger import Replay, hot_model, random_settings

gpu = pytest.mark.gpu
CHUNK = 1024


def _mod():
    import mycroft_precise_b200 as m
    return m


def same(x, y):
    x, y = np.ascontiguousarray(x), np.ascontiguousarray(y)
    return x.shape == y.shape and np.array_equal(x.view(np.uint8), y.view(np.uint8))


def activations(state, M=1):
    return state[:, 64:96].cpu().numpy().view(np.int32)[:, :M]


def continue_both(a, b, src, dst, rs, K, tick='update', chunk=CHUNK):
    """K ticks of the same items in the same order: a's streams src[j] and b's dst[j].  Every tick permutes the items; every
    third takes a partial set.  Returns a's outputs per tick (sids in a's ids)."""
    outs = []
    for k in range(K):
        j = rs.permutation(len(src))
        if k % 3 == 2:
            j = j[:len(src) // 2 + 1]
        pcm = noise((len(j), chunk), rs)
        oa = host(getattr(a, tick)(cuda(pcm), cuda(src[j])))
        ob = host(getattr(b, tick)(cuda(pcm), cuda(dst[j])))
        for x, y in zip(oa, ob):
            assert same(x, y), (tick, k)
        outs.append((src[j], oa))
    return outs


def prime(sb, rs, S, K, chunk=CHUNK):
    for k in range(K):
        sids = rs.permutation(S)[:S if k % 2 == 0 else S // 2 + 1].astype(np.int32)
        sb.update(cuda(noise((len(sids), chunk), rs)), cuda(sids))


@gpu
@pytest.mark.parametrize('S', [7, 9000])
def test_continuation_into_a_larger_handle(S):
    """A hot model primed with permuted, partial ticks; most of its streams move to other ids of a handle with more streams.
    B's windows equal A's right after the import, exporting them from B gives the imported bytes back, and the next ticks
    are bit-identical (9 000: the bank-kernel scan on full ticks, the warp kernel on partial ones).  4096-sample chunks and
    trigger level 1 (refractory -2: one quiet tick ends it; two hot ticks fire), so that streams imported in refractory fire
    again within the test (asserted at 9 000 streams)."""
    m = _mod()
    rs = np.random.RandomState(S)
    model = hot_model(m)
    chunk = 4096
    a, b = (m.StreamBatch(model, n, chunk_samples=chunk, trigger_level=1) for n in (S, S + 500))
    prime(a, rs, S, 12, chunk)
    src = rs.permutation(S)[:S - max(1, S // 20)].astype(np.int32)
    dst = rs.permutation(S + 500)[:len(src)].astype(np.int32)
    for k in range(48):                                                # until some exported stream is in refractory
        state = a.core.export_streams(cuda(src))
        act = activations(state)[:, 0]
        if (act < 0).any() and (S < 100 or (act > 0).any()):
            break
        prime(a, rs, S, 1, chunk)
    print('activations after %d more ticks: %d negative, %d positive of %d' % (k, (act < 0).sum(), (act > 0).sum(), len(act)))
    assert (act < 0).any() and (S < 100 or (act > 0).any())
    assert tuple(state.shape) == (len(src), a.core.stream_state_bytes) and a.core.stream_state_bytes % 16 == 0
    b.core.import_streams(state, dst)
    assert same(a.core.read_window(ids=cuda(src)).cpu().numpy(), b.core.read_window(ids=cuda(dst)).cpu().numpy())
    assert same(b.core.export_streams(cuda(dst)).cpu().numpy(), state.cpu().numpy())
    a.reset_count()
    b.reset_count()
    refr, fired_refr = set(src[act < 0].tolist()), set()
    for k in range(12):                                                # 4 ticks at a time until a refractory stream fires
        for sids, o in continue_both(a, b, src, dst, rs, 4, chunk=chunk):
            fired_refr |= set(sids[o[2].astype(bool)].tolist()) & refr
        if fired_refr and k >= 3:
            break
    assert int(a.count.item()) == int(b.count.item())
    if S >= 100:                                                       # seven streams of noise rarely fire within the test
        assert int(a.count.item()) > 0 and fired_refr, 'no stream imported in refractory fired afterwards'
    for x in (a, b):
        x.core.close()


@gpu
def test_checkpoint_through_disk_and_clear(tmp_path):
    """A checkpoint saved with np.save, A cleared, the checkpoint loaded and imported back: A continues as its twin that was
    never cleared.  The twin exports between every tick and must equal a third handle that never exports."""
    m = _mod()
    S = 300
    rs = np.random.RandomState(4)
    model = hot_model(m, seed=3)
    a, twin, plain = (m.StreamBatch(model, S) for _ in range(3))
    ticks = [(rs.permutation(S)[:S if k % 2 else 200].astype(np.int32), noise((S if k % 2 else 200, CHUNK), rs))
             for k in range(24)]

    def step(k):
        outs = []
        for x in (a, twin, plain):
            sids, pcm = ticks[k]
            outs.append(host(x.update(cuda(pcm), cuda(sids))))
        twin.core.export_streams(cuda(rs.permutation(S)[:50].astype(np.int32)))
        return outs

    for k in range(12):
        step(k)
    path = str(tmp_path / 'ckpt.npy')
    np.save(path, a.core.export_streams().cpu().numpy())
    a.core.clear()
    assert not a.core.export_streams()[:, 48:56].any().item()
    a.core.import_streams(cuda(np.load(path)))
    for k in range(12, 24):
        oa, ot, op = step(k)
        for x, y, z in zip(oa, ot, op):
            assert same(x, y) and same(y, z), k
    assert int(a.count.item()) == int(plain.count.item()) and int(twin.count.item()) == int(plain.count.item())
    assert same(a.core.export_streams().cpu().numpy(), plain.core.export_streams().cpu().numpy())
    for x in (a, twin, plain):
        x.core.close()


@gpu
@pytest.mark.parametrize('mode', ['force_generic', 'n_fft256', 'speechpy'])
def test_geometries(mode):
    """The generic K1, n_fft 256 and the speechpy vectoriser: continuation bit for bit, as in the first test."""
    m = _mod()
    pr = {'force_generic': m.ListenerParams(), 'n_fft256': m.ListenerParams(n_fft=256),
          'speechpy': m.ListenerParams(vectorizer=3)}[mode]
    S = 60
    rs = np.random.RandomState(9)
    model = m.GruModel.random(pr.feature_size, 20, seed=2, scale=0.1)
    model.dense_b = 3.0
    a, b = m.StreamBatch(model, S, params=pr), m.StreamBatch(model, S + 40, params=pr)
    if mode == 'force_generic':
        for x in (a, b):
            x.core.force_generic(True)
    prime(a, rs, S, 9)
    src = rs.permutation(S)[:50].astype(np.int32)
    dst = rs.permutation(S + 40)[:50].astype(np.int32)
    b.core.import_streams(a.core.export_streams(cuda(src)), dst)
    assert same(a.core.read_window(ids=cuda(src)).cpu().numpy(), b.core.read_window(ids=cuda(dst)).cpu().numpy())
    continue_both(a, b, src, dst, rs, 8)
    for x in (a, b):
        x.core.close()


@gpu
def test_other_chunk_size_follows_oracle():
    """A destination with chunk_samples 768 continues streams a 1024-sample source started: raw and conf against oracle
    Listeners fed the same audio, at the tolerances of smoke() and the parity tests."""
    from oracle.decoder import OracleDecoder
    from oracle.gru import GruWeights
    from oracle.listener import OracleListener
    from oracle.params import OracleParams
    m = _mod()
    S, K1, K2 = 5, 6, 10
    rs = np.random.RandomState(21)
    model = m.GruModel.random(13, 20, seed=1, scale=0.1)
    a, b = m.StreamBatch(model, S), m.StreamBatch(model, S, chunk_samples=768)
    audio = noise((S, K1 * 1024 + K2 * 768), rs)
    for k in range(K1):
        a.update(cuda(audio[:, k * 1024:(k + 1) * 1024]))
    b.core.import_streams(a.core.export_streams(), np.arange(S, dtype=np.int32)[::-1].copy())
    got = []
    for k in range(K2):
        lo = K1 * 1024 + k * 768
        got.append(host(b.update(cuda(audio[::-1, lo:lo + 768].copy()))))
    w = GruWeights(model.kernel, model.recurrent, model.bias, model.dense_w, model.dense_b)
    d = OracleDecoder(OracleParams().threshold_config, OracleParams().threshold_center)
    step = float(np.max(np.abs(np.diff(d.cd)))) * 2.5
    for s in range(S):
        lis = OracleListener(w, OracleParams())
        for k in range(K1):
            lis.update_raw(audio[s, k * 1024:(k + 1) * 1024].astype(np.float32) / 32768.0)
        for k in range(K2):
            lo = K1 * 1024 + k * 768
            r = lis.update_raw(audio[s, lo:lo + 768].astype(np.float32) / 32768.0)
            raw, conf = got[k][0][S - 1 - s], got[k][1][S - 1 - s]
            assert abs(raw - r) < 1e-4 and abs(conf - lis.decoder.decode(r)) <= step, (s, k, raw, r)
    for x in (a, b):
        x.core.close()


def ragged_ticks(sb, rs, S, K):
    for k in range(K):
        sids = rs.permutation(S).astype(np.int32)
        lens = rs.randint(600, 1500, S)
        offs = cuda((1 + np.concatenate([[0], np.cumsum(lens)])).astype(np.int64))
        sb.update_ragged(cuda(noise((int(lens.sum()) + 1,), rs)), offs, cuda(sids), max_len=1500)


@gpu
def test_ragged_rule():
    """Records with n_samples % 8 != 0 make a fresh fast-geometry handle ragged (k1 mode 2 is refused afterwards) and continue
    bit for bit; a destination in k1 mode 2 refuses them and is unchanged; aligned records leave k1 mode 2 available."""
    m = _mod()
    S = 40
    rs = np.random.RandomState(31)
    model = hot_model(m, seed=9)
    a = m.StreamBatch(model, S)
    ragged_ticks(a, rs, S, 6)
    state = a.core.export_streams()
    ns = state[:, 48:56].cpu().numpy().view(np.int64)[:, 0]
    assert (ns % 8 != 0).any()
    ids = np.arange(S, dtype=np.int32)
    fast = m.StreamBatch(model, S)
    fast.core.k1_mode(2)
    before = fast.core.export_streams().cpu().numpy()
    with pytest.raises(m.PBError):
        fast.core.import_streams(state, ids)
    assert same(fast.core.export_streams().cpu().numpy(), before)
    fast.core.k1_mode(0)
    b = m.StreamBatch(model, S)
    b.core.import_streams(state, ids)
    with pytest.raises(m.PBError):
        b.core.k1_mode(2)
    continue_both(a, b, ids, ids, rs, 6)
    aligned = m.StreamBatch(model, S)
    prime(aligned, rs, S, 4)
    fast.core.import_streams(aligned.core.export_streams(), ids)
    fast.core.k1_mode(2)
    continue_both(aligned, fast, ids, ids, rs, 4)
    for x in (a, b, fast, aligned):
        x.core.close()


@gpu
def test_bank_with_masks_and_settings():
    """The four-model bank, routed, with trigger settings on slots 0 and 2, moved with StreamBatch.export_streams /
    import_streams: masks and settings read back equal, update_models and update_ragged continue bit for bit, and fired
    follows the oracle TriggerDetector replayed over the source's conf from its first tick."""
    m = _mod()
    S, S2 = 2000, 2600
    rs = np.random.RandomState(41)
    spec = bank_models(m)
    a, b = bank(m, spec, S), bank(m, spec, S2)
    rep = Replay(spec)
    mask = rs.randint(0, 256, S).astype(np.uint8)
    a.set_stream_models(mask)
    for mi in (0, 2):
        ids = rs.permutation(S)[:S - 200].astype(np.int32)
        sens, lvl, chunk = random_settings(rs, len(ids), (0.1, 0.4, 0.6))
        a.set_stream_trigger(mi, sens, lvl, chunk, ids=ids)
        rep.set(mi, ids, sens, lvl, chunk)
    for k in range(8):
        sids = rs.permutation(S)[:S if k % 2 else S // 2].astype(np.int32)
        rep.tick(sids, host(a.update_models(cuda(noise((len(sids), CHUNK), rs)), cuda(sids))), None, mask)
    src = rs.permutation(S)[:1800].astype(np.int32)
    dst = rs.permutation(S2)[:1800].astype(np.int32)
    snap = a.export_streams(src)
    snap['state'] = snap['state'].cpu()
    b.import_streams(snap, dst)
    assert np.array_equal(b.core.stream_models(dst), a.core.stream_models(src))
    for mi in range(4):
        for x, y in zip(b.stream_trigger(mi, dst), a.stream_trigger(mi, src)):
            assert same(x, y), mi
    a.reset_count()
    b.reset_count()
    fired = np.zeros(4, np.int64)
    for k in range(10):
        j = rs.permutation(len(src))[:1800 if k % 3 else 900]
        if k % 2 == 0:
            pcm = cuda(noise((len(j), CHUNK), rs))
            oa, ob = host(a.update_models(pcm, cuda(src[j]))), host(b.update_models(pcm, cuda(dst[j])))
        else:
            lens = rs.randint(700, 1400, len(j))
            offs = cuda((3 + np.concatenate([[0], np.cumsum(lens)])).astype(np.int64))
            pcm = cuda(noise((int(lens.sum()) + 5,), rs))
            oa = host(a.update_ragged(pcm, offs, cuda(src[j]), max_len=1400))
            ob = host(b.update_ragged(pcm, offs, cuda(dst[j]), max_len=1400))
        for x, y in zip(oa, ob):
            assert same(x, y), k
        rep.tick(src[j], oa, None, mask)
        fired += oa[2].sum(axis=1).astype(np.int64)
    assert np.array_equal(a.counts.cpu().numpy(), b.counts.cpu().numpy()) and np.array_equal(b.counts.cpu().numpy(), fired)
    print('fired per model', fired)
    assert fired[[0, 2]].min() > 0
    for x in (a, b):
        x.core.close()


@gpu
def test_validation_changes_nothing():
    m = _mod()
    S = 1200
    rs = np.random.RandomState(51)
    model = hot_model(m, seed=2)
    a, b = m.StreamBatch(model, S), m.StreamBatch(model, S)
    prime(a, rs, S, 4)
    prime(b, rs, S, 3)
    b.set_stream_models(np.full(S, 1, np.uint8))
    good = a.core.export_streams()
    B = a.core.stream_state_bytes
    lib, h = b.core.lib, b.core._h
    ids = np.arange(S, dtype=np.int32)

    def snapshot():
        return b.core.export_streams().cpu().numpy(), b.core.stream_models()

    want = snapshot()

    def refuse(state, n=None, idv=ids, rc=-1, what=None, ptr=None):
        n = state.shape[0] if n is None else n
        p = C.c_void_p(state.data_ptr()) if ptr is None else ptr
        got = lib.pb_import_streams(h, None if idv is None else idv.ctypes.data_as(C.c_void_p), n, p)
        msg = lib.pb_last_error().decode()
        assert got == rc, (got, msg)
        if what:
            assert what in msg, msg
        now = snapshot()
        assert same(now[0], want[0]) and np.array_equal(now[1], want[1])

    bad = good[:1000].clone()
    bad[617, 48:56] = cuda(np.array([-8], np.int64).view(np.uint8))            # one bad record among 1 000
    refuse(bad, idv=ids[:1000], what='record 617')
    for off, what in ((0, 'magic'), (4, 'version')):
        bad = good[:5].clone()
        bad[3, off] ^= 1
        refuse(bad, idv=ids[:5], what=what)
    other = m.StreamBatch(m.GruModel.random(13, 20, seed=1, scale=0.1), 4, params=m.ListenerParams(n_fft=256))
    rec = other.core.export_streams()
    assert other.core.stream_state_bytes < B
    bad = good[:4].clone()
    bad[:, :rec.shape[1]] = rec
    refuse(bad, idv=ids[:4], what='n_fft')
    two = bank(m, [(model, None, 0.5, 3), (model, None, 0.5, 3)], 4)
    refuse(two.core.export_streams(), idv=ids[:4], what='num_models')
    refuse(good[:3], idv=np.array([1, 2, 1], np.int32), what='twice')
    refuse(good[:3], idv=np.array([1, 2, S], np.int32))
    refuse(good[:3], idv=np.array([-1, 2, 3], np.int32))
    refuse(good, n=-1, idv=None)
    refuse(good, n=S + 1, idv=None)
    refuse(good, n=3, idv=None, ptr=C.c_void_p(0), what='null')
    refuse(good, n=3, idv=None, ptr=C.c_void_p(good.data_ptr() + 8), what='aligned')
    assert lib.pb_export_streams(h, None, 3, C.c_void_p(good.data_ptr() + 8), None) == -1
    assert lib.pb_export_streams(h, None, S + 1, C.c_void_p(good.data_ptr()), None) == -1
    for case in (good[:, :-16], good.view(b.core.torch.int32), good.cpu(), good[:3].flatten()):
        with pytest.raises(ValueError):
            b.core.import_streams(case)
    with pytest.raises(ValueError):
        b.core.import_streams(good[:3], ids=np.array([0, 1], np.int32))
    with pytest.raises(ValueError):
        b.core.export_streams(n=3, out=good[:2])
    snap = two.export_streams()
    snap['stream_trigger'] = snap['stream_trigger'][:1]
    snap['stream_models'] = np.zeros(4, np.uint8)
    with pytest.raises(ValueError, match='num_models'):
        b.import_streams(snap)
    now = snapshot()
    assert same(now[0], want[0]) and np.array_equal(now[1], want[1])
    b.core.k1_mode(2)                                                          # no import above made b ragged
    for x in (a, b, other, two):
        x.core.close()


@gpu
def test_cross_device():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two GPUs')
    m = _mod()
    S = 100
    rs = np.random.RandomState(61)
    model = hot_model(m, seed=5)
    a, b = m.StreamBatch(model, S, device=0), m.StreamBatch(model, S, device=1)
    prime(a, rs, S, 6)
    b.core.import_streams(a.core.export_streams().to('cuda:1'))
    for k in range(6):
        pcm = noise((S, CHUNK), rs)
        oa = host(a.update(torch.from_numpy(pcm).to('cuda:0')))
        ob = host(b.update(torch.from_numpy(pcm).to('cuda:1')))
        for x, y in zip(oa, ob):
            assert same(x, y), k
    for x in (a, b):
        x.core.close()


def test_stream_state_null_handle_is_invalid():
    import os
    import __graft_entry__ as g
    from mycroft_precise_b200.core import lib_path, get_lib
    if not os.path.isfile(lib_path()):
        g.build()
    lib = get_lib()
    buf = np.zeros(64, np.uint8)
    p = buf.ctypes.data_as(C.c_void_p)
    assert lib.pb_stream_state_bytes(None) == -1 and b'null' in lib.pb_last_error()
    assert lib.pb_export_streams(None, None, 1, p, None) == -1
    assert lib.pb_export_streams(None, None, 0, None, None) == -1
    assert lib.pb_import_streams(None, None, 1, p) == -1
    assert lib.pb_import_streams(None, None, 0, None) == -1
