"""Per-stream model subscriptions (pb_set_stream_models): routed bank ticks, the slot-0 paths and their edge cases.

-m gpu, except the C-ABI null-handle check at the end.  A routed handle must score every subscribed (stream, model) pair
bit-identically to an identical handle that never sets masks, return NaN / NaN / 0 for every other pair, and run each model's
TriggerDetector only over the ticks its stream is subscribed to, re-armed when the stream's bit goes from 0 to 1 and at a clear.
"""
import ctypes as C

import numpy as np
import pytest

from oracle.trigger import OracleTrigger
from test_gpu_model_bank import bank_models

gpu = pytest.mark.gpu
CHUNK = 1024


def _mod():
    import mycroft_precise_b200 as m
    return m


def cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def noise(shape, rs, sigma=3000):
    return np.clip(rs.randn(*shape) * sigma, -32768, 32767).astype(np.int16)


def bank(m, spec, S):
    sb = m.StreamBatch(spec[0][0], S, params=spec[0][1], sensitivity=spec[0][2], trigger_level=spec[0][3])
    for model, pr, sens, lvl in spec[1:]:
        sb.add_model(model, pr, sensitivity=sens, trigger_level=lvl)
    return sb


def host(o):
    return o['raw'].cpu().numpy(), o['conf'].cpu().numpy(), o['fired'].cpu().numpy()


class Checker:
    """Checks a routed tick against the masks, the unrouted handle's outputs and the oracle trigger replayed on the routed
    handle's own conf over the subscribed ticks only."""

    def __init__(self, spec):
        self.trig = [(sens, lvl) for _, _, sens, lvl in spec]
        self.det = {}
        self.fired = np.zeros(len(spec), np.int64)

    def set_masks(self, old, new, sids):
        for sid in sids:
            for mi in range(8):
                if (new[sid] >> mi) & 1 and not (old[sid] >> mi) & 1:
                    self.det.pop((int(sid), mi), None)          # 0 -> 1: a new detector

    def clear(self, sids):
        for sid in sids:
            for mi in range(8):
                self.det.pop((int(sid), mi), None)

    def tick(self, mask, sids, a, b=None):
        """a = routed (raw, conf, fired), b = unrouted (raw, conf) or None; each [M, n]."""
        ra, ca, fa = (np.asarray(x).reshape(-1, len(sids)) for x in a)
        M = ra.shape[0]
        sub = ((mask[sids][None, :] >> np.arange(M)[:, None]) & 1).astype(bool)
        if b is not None:
            rb, cb = (np.asarray(x).reshape(M, -1) for x in b)
            bad_r = int(np.sum(ra[sub].view(np.uint32) != rb[sub].view(np.uint32)))
            bad_c = int(np.sum(ca[sub].view(np.uint64) != cb[sub].view(np.uint64)))
            assert bad_r == 0 and bad_c == 0, 'subscribed pairs differ from the unrouted handle: raw %d, conf %d of %d' % (
                bad_r, bad_c, int(sub.sum()))
        assert np.isnan(ra[~sub]).all() and np.isnan(ca[~sub]).all() and not fa[~sub].any(), 'unsubscribed pairs not NaN / NaN / 0'
        for mi, j in zip(*np.nonzero(sub)):
            key = (int(sids[j]), int(mi))
            if key not in self.det:
                self.det[key] = OracleTrigger(CHUNK * 2, *self.trig[mi])
            assert bool(fa[mi, j]) == self.det[key].update(float(ca[mi, j])), key
        self.fired[:M] += fa.sum(axis=1).astype(np.int64)
        return sub


@gpu
@pytest.mark.parametrize('S', [7, 9000])
def test_routed_bank_equals_unrouted_bank(S):
    """The four-model bank (H = 32 outside the fused family, a tanh / sigmoid model), random masks including 0 and 0xFF,
    permuted and partial ticks, mask changes between ticks and a clear."""
    m = _mod()
    rs = np.random.RandomState(S)
    spec = bank_models(m)
    a, b = bank(m, spec, S), bank(m, spec, S)
    mask = rs.randint(0, 256, S).astype(np.uint8)
    mask[0], mask[1] = 0, 0xFF
    a.set_stream_models(mask)
    assert np.array_equal(a.core.stream_models(), mask)
    chk = Checker(spec)
    for k in range(14):
        if k in (5, 10):                                              # some streams change masks
            sel = rs.choice(S, max(2, S // 3), replace=False).astype(np.int32)
            new = mask.copy()
            new[sel] = rs.randint(0, 256, len(sel))
            new[sel[0]] = mask[sel[0]] ^ 0xFF
            a.set_stream_models(new[sel], sel)
            chk.set_masks(mask, new, sel)
            mask = new
        if k == 8:
            cl = np.sort(rs.choice(S, max(1, S // 4), replace=False)).astype(np.int32)
            a.clear(cuda(cl))
            b.clear(cuda(cl))
            chk.clear(cl)
        kind = k % 3
        if kind == 0:
            sids, ids = np.arange(S), None
        else:
            sids = rs.permutation(S)[:S if kind == 1 else S // 2 + 1].astype(np.int32)
            ids = cuda(sids)
        c = cuda(noise((len(sids), CHUNK), rs))
        oa = host(a.update_models(c, ids))
        ob = host(b.update_models(c, ids))
        chk.tick(mask, sids, oa, ob[:2])
    counts = a.counts.cpu().numpy()
    print('fired per model', chk.fired, 'counts', counts)
    assert np.array_equal(counts, chk.fired)
    for x in (a, b):
        x.core.close()


@gpu
def test_one_model_per_stream_at_scale():
    """8 fused models (five with Keras's default activations, three with other pairs), 20 000 streams, stream s on model s mod 8:
    each model's outputs equal a one-model handle's bank tick of that model on the same audio, bit for bit."""
    m = _mod()
    S, K = 20000, 5
    rs = np.random.RandomState(3)
    acts = [('linear', 'hard_sigmoid')] * 5 + [('tanh', 'sigmoid'), ('linear', 'sigmoid'), ('tanh', 'hard_sigmoid')]
    models = []
    for i, (H, (ac, ra)) in enumerate(zip([20, 12, 24, 16, 20, 20, 8, 24], acts)):
        mod = m.GruModel.random(13, H, seed=40 + i, scale=0.1)
        mod.activation, mod.recurrent_activation = ac, ra
        models.append(mod)
    routed = bank(m, [(mod, None, 0.5, 3) for mod in models], S)
    mask = (1 << (np.arange(S) % 8)).astype(np.uint8)
    routed.set_stream_models(mask)
    solo = [m.StreamBatch(mod, S) for mod in models]
    chk = Checker([(mod, None, 0.5, 3) for mod in models])
    for k in range(K):
        c = cuda(noise((S, CHUNK), rs))
        o = host(routed.update_models(c))
        chk.tick(mask, np.arange(S), o)
        for i, sb in enumerate(solo):
            r, cf, _ = host(sb.update_models(c))
            sel = np.arange(S) % 8 == i
            assert np.array_equal(o[0][i, sel].view(np.uint32), r[0, sel].view(np.uint32)), (k, i)
            assert np.array_equal(o[1][i, sel].view(np.uint64), cf[0, sel].view(np.uint64)), (k, i)
    assert np.array_equal(routed.counts.cpu().numpy(), chk.fired)
    for x in [routed] + solo:
        x.core.close()


@gpu
def test_slot0_paths():
    """A one-model routed handle: update at n <= 8 192 (warp per stream) and above (the bank kernel), the CUDA-core kernel
    (gru mode 1) and update_host; unsubscribed streams later resubscribe and their triggers follow the oracle."""
    m = _mod()
    S = 9000
    rs = np.random.RandomState(11)
    model = m.GruModel.random(13, 20, seed=8, scale=0.1)
    model.dense_b = 3.0                                                # confidences often over the trigger threshold
    spec = [(model, None, 0.5, 3)]
    a, b = bank(m, spec, S), bank(m, spec, S)
    mask = (rs.randint(0, 2, S) | (rs.randint(0, 128, S) << 1)).astype(np.uint8)
    a.set_stream_models(mask)
    chk = Checker(spec)
    host_count = 0
    plan = ['small', 'big', 'host', 'small', 'mode1', 'big', 'host_part', 'resub', 'small', 'big', 'host', 'big']
    for what in plan:
        if what == 'resub':
            new = mask | 1
            a.set_stream_models(new)
            chk.set_masks(mask, new, np.arange(S))
            mask = new
            continue
        if what in ('host', 'host_part'):
            sids = np.arange(S, dtype=np.int32) if what == 'host' else np.sort(rs.permutation(S)[:5000]).astype(np.int32)
            pcm = noise((len(sids), CHUNK), rs)
            outs = []
            for x in (a, b):
                raw, conf, fired = np.zeros(len(sids), np.float32), np.zeros(len(sids)), np.zeros(len(sids), np.uint8)
                cnt = x.core.update_host(pcm, conf, raw, fired, None if what == 'host' else sids)
                outs.append((raw, conf, fired, cnt))
            chk.tick(mask, sids, outs[0][:3], outs[1][:2])
            assert outs[0][3] == int(outs[0][2].sum())
            host_count += outs[0][3]
            continue
        sids = rs.permutation(S)[:5000].astype(np.int32) if what == 'small' else np.arange(S, dtype=np.int32)
        if what == 'mode1':
            for x in (a, b):
                x.core.gru_mode(1)
        c, ids = cuda(noise((len(sids), CHUNK), rs)), cuda(sids)
        oa, ob = host(a.update(c, ids)), host(b.update(c, ids))
        chk.tick(mask, sids, oa, ob[:2])
        if what == 'mode1':
            for x in (a, b):
                x.core.gru_mode(0)
    print('fired', chk.fired, 'count', int(a.count.item()), 'host ticks', host_count)
    assert int(a.count.item()) + host_count == chk.fired[0] and chk.fired[0] > 0
    for x in (a, b):
        x.core.close()


@gpu
def test_ragged_ticks_on_routed_bank():
    m = _mod()
    import torch
    S = 3000
    rs = np.random.RandomState(21)
    spec = bank_models(m)
    a, b = bank(m, spec, S), bank(m, spec, S)
    mask = rs.randint(0, 256, S).astype(np.uint8)
    a.set_stream_models(mask)
    chk = Checker(spec)
    for k in range(10):
        sids = (np.arange(S) if k % 2 == 0 else rs.permutation(S)[:2000]).astype(np.int32)
        lens = rs.randint(500, 1500, len(sids))
        offs = cuda(np.concatenate([[0], np.cumsum(lens)]).astype(np.int64))
        pcm = cuda(noise((int(lens.sum()),), rs))
        ids = cuda(sids)
        oa = host(a.update_ragged(pcm, offs, ids, max_len=1500))
        ob = host(b.update_ragged(pcm, offs, ids, max_len=1500))
        chk.tick(mask, sids, oa, ob[:2])
        if k == 4:
            new = rs.randint(0, 256, S).astype(np.uint8)
            a.set_stream_models(new)
            chk.set_masks(mask, new, np.arange(S))
            mask = new
    torch.cuda.synchronize()
    assert np.array_equal(a.counts.cpu().numpy(), chk.fired)
    for x in (a, b):
        x.core.close()


@gpu
def test_edge_cases():
    """A fused and a non-fused model without subscribers (all NaN); streams with mask 0 keep their MFCC state and later
    subscribe; a model added after the masks were set scores exactly the streams whose mask has its slot's bit."""
    m = _mod()
    S = 500
    rs = np.random.RandomState(5)
    spec = bank_models(m)
    a, b = bank(m, spec, S), bank(m, spec, S)
    mask = (rs.randint(0, 256, S) & ~0b1010).astype(np.uint8)          # models 1 (H = 12) and 3 (H = 32): nobody
    mask[:50] = 0
    a.set_stream_models(mask)
    chk = Checker(spec)
    for k in range(4):
        c = cuda(noise((S, CHUNK), rs))
        oa, ob = host(a.update_models(c)), host(b.update_models(c))
        chk.tick(mask, np.arange(S), oa, ob[:2])
        assert np.isnan(oa[0][[1, 3]]).all() and np.isnan(oa[1][[1, 3]]).all() and not oa[2][[1, 3]].any()
    wa, wb = a.core.read_window(S).cpu().numpy(), b.core.read_window(S).cpu().numpy()
    assert np.array_equal(wa.view(np.uint32), wb.view(np.uint32))
    new = mask.copy()
    new[:50] = 0xFF
    a.set_stream_models(new[:50], np.arange(50, dtype=np.int32))
    chk.set_masks(mask, new, np.arange(50))
    mask = new
    for k in range(3):
        c = cuda(noise((S, CHUNK), rs))
        chk.tick(mask, np.arange(S), host(a.update_models(c)), host(b.update_models(c))[:2])
    assert np.array_equal(a.counts.cpu().numpy(), chk.fired)
    for x in (a, b):
        x.core.close()

    # pb_add_model after the masks are set
    a, b = bank(m, spec[:1], S), bank(m, spec[:1], S)
    mask = np.full(S, 0xFF, np.uint8)
    mask[100:200] = 0x01                                               # narrowed to slot 0
    mask[200:300] = 0x04                                               # narrowed to a slot not yet added
    mask[300:320] = 0x00
    a.set_stream_models(mask[100:320], np.arange(100, 320, dtype=np.int32))
    chk = Checker(spec[:2])
    for k in range(3):
        c = cuda(noise((S, CHUNK), rs))
        chk.tick(mask, np.arange(S), host(a.update(c)), host(b.update(c))[:2])
    for x in (a, b):
        x.add_model(spec[1][0], spec[1][1], sensitivity=spec[1][2], trigger_level=spec[1][3])
    for k in range(3):
        c = cuda(noise((S, CHUNK), rs))
        oa = host(a.update_models(c))
        sub = chk.tick(mask, np.arange(S), oa, host(b.update_models(c))[:2])
        assert np.array_equal(np.nonzero(sub[1])[0], np.r_[0:100, 320:S])
    assert int(a.count.item()) + int(a.counts[0].item()) == chk.fired[0] and int(a.counts[1].item()) == chk.fired[1]
    for x in (a, b):
        x.core.close()


@gpu
def test_stream_models_errors():
    m = _mod()
    c = m.PreciseB200(max_streams=16)
    assert c.stream_models().dtype == np.uint8 and np.all(c.stream_models() == 0xFF)
    bad = [(np.ones(2, np.uint8), np.array([3, 16], np.int32)),                # id out of range
           (np.ones(2, np.uint8), np.array([3, -1], np.int32)),
           (np.ones(2, np.uint8), np.array([3, 3], np.int32)),                 # duplicate id
           (np.ones(17, np.uint8), None),                                      # n > max_streams
           (np.ones(2, np.int64), None)]                                       # not uint8
    for masks, ids in bad:
        with pytest.raises(ValueError):
            c.set_stream_models(masks, ids)
    assert np.all(c.stream_models() == 0xFF)
    c.set_stream_models(np.array([5, 0], np.uint8), np.array([2, 9], np.int32))
    want = np.full(16, 0xFF, np.uint8)
    want[2], want[9] = 5, 0
    for masks, ids in bad:
        with pytest.raises(ValueError):
            c.set_stream_models(masks, ids)
    assert np.array_equal(c.stream_models(), want)
    assert np.array_equal(c.stream_models(np.array([9, 2], np.int32)), [0, 5])
    with pytest.raises(ValueError):
        c.stream_models(np.array([16], np.int32))
    n = np.ones(17, np.uint8)
    assert c.lib.pb_set_stream_models(c._h, None, n.ctypes.data_as(C.c_void_p), 17) == -1
    assert c.lib.pb_get_stream_models(c._h, None, 17, n.ctypes.data_as(C.c_void_p)) == -1
    c.close()


def test_stream_models_null_handle_is_invalid():
    import os
    import __graft_entry__ as g
    from mycroft_precise_b200.core import lib_path, get_lib
    if not os.path.isfile(lib_path()):
        g.build()
    lib = get_lib()
    masks = np.zeros(4, np.uint8)
    ids = np.arange(4, dtype=np.int32)
    p, q = masks.ctypes.data_as(C.c_void_p), ids.ctypes.data_as(C.c_void_p)
    assert lib.pb_set_stream_models(None, q, p, 4) == -1 and b'null' in lib.pb_last_error()
    assert lib.pb_get_stream_models(None, q, 4, p) == -1
    assert lib.pb_set_stream_models(None, None, None, 0) == -1
