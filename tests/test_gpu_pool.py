"""Model pool (pb_set_pool / pb_pool_load / pb_set_stream_pool / pb_update_pool, pool.cuh): each stream scored by at most one
of many networks of the fused family.

The reference for every pool stream is the same network in an unrouted bank over the same streams and audio: raw and conf
must be equal bit for bit.  fired is checked against OracleTrigger replayed on the pool's own conf, with a fresh detector
wherever the stream's model changed, it was cleared or its model was reloaded.  -m gpu, except the null-handle check."""
import ctypes as C

import numpy as np
import pytest

from oracle import gru as og
from oracle.trigger import OracleTrigger

gpu = pytest.mark.gpu
CHUNK = 1024


def _mod():
    import mycroft_precise_b200 as m
    return m


def cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def noise(S, L, seed=0, sigma=3000):
    rs = np.random.RandomState(seed)
    return np.clip(rs.randn(S, L) * sigma, -32768, 32767).astype(np.int16)


def pool_models(m):
    """(model, params, sensitivity, trigger_level) of twelve fused networks: the fused models of the bank tests (the default
    network, H = 12 with its own decoder and trigger, tanh / sigmoid) and seeded variants.  Dense biases make them fire."""
    m0 = m.GruModel.random(13, 20, seed=0, scale=0.1)
    m1 = m.GruModel.random(13, 12, seed=1, scale=0.1)
    m2 = m.GruModel.random(13, 20, seed=2, scale=0.1)
    m2.activation, m2.recurrent_activation = 'tanh', 'sigmoid'
    p1 = m.ListenerParams(threshold_config=((8, 3),), threshold_center=0.3)
    spec = [(m0, None, 0.8, 1), (m1, p1, 0.8, 1), (m2, None, 0.5, 3)]
    for i in range(9):
        g = m.GruModel.random(13, [20, 12, 24, 16, 8][i % 5], seed=100 + i, scale=0.1)
        if i % 3 == 2:
            g.activation, g.recurrent_activation = 'tanh', 'sigmoid'
        spec.append((g, None, 0.5 + 0.1 * (i % 4), 1 + i % 3))
    for i, (g, pr, _, _) in enumerate(spec):
        g.dense_b = (pr.threshold_config[0][0] if pr is not None else 3.0) - 0.5 * (i % 3)
    return spec


def banks_of(m, spec, S):
    """Two unrouted banks of six: model i is slot i % 6 of bank i // 6."""
    out = []
    for b in range(0, len(spec), 6):
        part = spec[b:b + 6]
        sb = m.StreamBatch(part[0][0], S, params=part[0][1], chunk_samples=CHUNK, sensitivity=part[0][2],
                           trigger_level=part[0][3])
        for model, pr, sens, lvl in part[1:]:
            sb.add_model(model, pr, sensitivity=sens, trigger_level=lvl)
        out.append(sb)
    return out


def pool_of(m, spec, S, models=None):
    sb = m.StreamBatch(spec[0][0], S, chunk_samples=CHUNK)
    sb.set_pool(len(spec) if models is None else models)
    for i, (model, pr, sens, lvl) in enumerate(spec):
        sb.pool_load(i, model, pr, sensitivity=sens, trigger_level=lvl)
    return sb


def assignment(S, n_models, seed):
    """Model of each stream: groups of 1, 15, 16, 17, 63, 64, 65 and about 200 (as far as S allows), the rest of the models
    sharing what is left; about 5 % of the streams on none.  Streams in random order."""
    unassigned = max(3, S // 20)
    avail = S - unassigned
    sizes = []
    for z in (1, 15, 16, 17, 63, 64, 65, 200):
        if sum(sizes) + z + (n_models - len(sizes) - 1) <= avail:
            sizes.append(z)
    left = n_models - len(sizes)
    rest = avail - sum(sizes)
    sizes += [rest // left + (1 if j < rest % left else 0) for j in range(left)]
    ids = np.concatenate([np.full(z, k, np.int32) for k, z in enumerate(sizes)] + [np.full(unassigned, -1, np.int32)])
    return np.random.RandomState(seed).permutation(ids).astype(np.int32)


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


class Replay:
    """OracleTrigger per stream, fresh when the stream's model changes, on clears and on reloads of its model."""

    def __init__(self, spec, S):
        self.spec, self.det = spec, [None] * S

    def rearm(self, sids):
        for s in np.atleast_1d(sids):
            self.det[int(s)] = None

    def check(self, sids, mids, conf, fired):
        want = np.zeros(len(sids), np.uint8)
        for j, (s, mid) in enumerate(zip(sids, mids)):
            if mid < 0:
                continue
            if self.det[s] is None:
                _, _, sens, lvl = self.spec[mid]
                self.det[s] = OracleTrigger(2 * CHUNK, sens, lvl)
            want[j] = self.det[s].update(float(conf[j]))
        assert np.array_equal(fired, want)
        return int(want.sum())


def check_tick(po, bank_out, sids, mids):
    """The pool's [n] outputs against the banks' rows: bit-identical raw and conf where the stream has a model, NaN / NaN /
    0 where it has none."""
    raw, conf, fired = (po[k].cpu().numpy() for k in ('raw', 'conf', 'fired'))
    R = np.concatenate([b['raw'] for b in bank_out])
    Cf = np.concatenate([b['conf'] for b in bank_out])
    on = mids >= 0
    j = np.nonzero(on)[0]
    assert np.array_equal(bits(raw[on]), bits(R[mids[on], j]))
    assert np.array_equal(bits(conf[on]), bits(Cf[mids[on], j]))
    assert np.isnan(raw[~on]).all() and np.isnan(conf[~on]).all() and not fired[~on].any()
    return raw, conf, fired


def run_banks(banks, pcm, ids=None, offsets=None, max_len=None):
    out = []
    for b in banks:
        o = b.update_models(pcm, ids) if offsets is None else b.update_ragged(pcm, offsets, ids, max_len)
        out.append({k: o[k].cpu().numpy().copy() for k in ('raw', 'conf')})
    return out


@gpu
@pytest.mark.parametrize('S', [300, 9000])
def test_pool_bit_identical_to_banks(S):
    m = _mod()
    spec = pool_models(m)
    assign = assignment(S, len(spec), seed=S)
    banks = banks_of(m, spec, S)
    pool = pool_of(m, spec, S)
    pool.set_stream_pool(assign)
    assert np.array_equal(pool.stream_pool(), assign)
    K = 12 if S == 300 else 8
    pcm = noise(S, K * CHUNK, seed=S + 1)
    rep = Replay(spec, S)
    fired_total = 0
    sids = np.arange(S, dtype=np.int32)
    for k in range(K):
        c = cuda(pcm[:, k * CHUNK:(k + 1) * CHUNK])
        bo = run_banks(banks, c)
        po = pool.update_pool(c)
        _, conf, fired = check_tick(po, bo, sids, assign)
        fired_total += rep.check(sids, assign, conf, fired)
    print('S = %d: %d pool fires' % (S, fired_total))
    assert fired_total > 0 and int(pool.pool_count.item()) == fired_total
    if S == 300:                     # spot check against the float64 network on the GPU's own windows
        wins = pool.core.read_window(S).cpu().numpy()
        raw = po['raw'].cpu().numpy()
        for mid, (model, _, _, _) in enumerate(spec):
            sel = assign == mid
            w = og.GruWeights(model.kernel, model.recurrent, model.bias, model.dense_w, model.dense_b,
                              model.activation, model.recurrent_activation)
            p64 = og.gru_forward(w, wins[sel], np.float64)[0].reshape(-1)
            assert np.max(np.abs(raw[sel] - p64)) < 1e-5
    for x in banks + [pool]:
        x.core.close()


@gpu
def test_pool_ticks_permuted_partial_ragged():
    """Full, permuted and partial ticks, ragged ticks with odd offsets and lengths (against the banks' update_ragged), and
    uniform ticks after them."""
    import torch
    m = _mod()
    S = 700
    spec = pool_models(m)
    assign = assignment(S, len(spec), seed=5)
    banks = banks_of(m, spec, S)
    pool = pool_of(m, spec, S)
    pool.set_stream_pool(assign)
    rs = np.random.RandomState(6)
    rep = Replay(spec, S)
    plan = ['full', 'perm', 'subset', 'full', 'ragged', 'subset', 'ragged', 'full', 'perm', 'full']
    for k, what in enumerate(plan):
        if what == 'ragged':
            sids = rs.permutation(S)[:S - 50].astype(np.int32)
            lens = rs.randint(1, 2 * CHUNK, size=sids.size)
            lens[::3] |= 1
            offs = np.concatenate([[3], 3 + np.cumsum(lens)]).astype(np.int64)
            flat = noise(1, int(offs[-1]), seed=100 + k)[0]
            pcm, offsets, ids = cuda(flat), cuda(offs), cuda(sids)
            max_len = int(lens.max())
            bo = run_banks(banks, pcm, ids, offsets, max_len)
            po = pool.update_pool(pcm, ids, offsets=offsets, max_len=max_len)
        else:
            if what == 'full':
                sids = np.arange(S, dtype=np.int32)
            elif what == 'perm':
                sids = rs.permutation(S).astype(np.int32)
            else:
                sids = np.sort(rs.choice(S, S // 3, replace=False)).astype(np.int32)
            pcm = cuda(noise(sids.size, CHUNK, seed=200 + k))
            ids = None if what == 'full' else cuda(sids)
            bo = run_banks(banks, pcm, ids)
            po = pool.update_pool(pcm, ids)
        _, conf, fired = check_tick(po, bo, sids, assign[sids])
        rep.check(sids, assign[sids], conf, fired)
    torch.cuda.synchronize()
    for x in banks + [pool]:
        x.core.close()


@gpu
def test_pool_changes_between_ticks():
    """Reassignments (to and from -1) re-arm, same-model sets keep the detector, clears re-arm, a reload switches the slot's
    streams to the new weights and re-arms them, and set_pool again unassigns every stream."""
    import torch
    m = _mod()
    S = 400
    spec = pool_models(m)[:6]
    banks = banks_of(m, spec, S)                 # one bank: model i is row i
    pool = m.StreamBatch(spec[0][0], S, chunk_samples=CHUNK)
    pool.set_pool(4)
    for i in range(4):
        pool.pool_load(i, spec[i][0], spec[i][1], sensitivity=spec[i][2], trigger_level=spec[i][3])
    rs = np.random.RandomState(9)
    assign = rs.randint(-1, 4, size=S).astype(np.int32)
    pool.set_stream_pool(assign)
    row = np.arange(6)                           # bank row of each pool slot (changes with the reload)
    rep = Replay(spec, S)
    sids = np.arange(S, dtype=np.int32)
    for k in range(16):
        if k == 4:                               # reassign some streams, set others to the model they have
            ch = rs.choice(S, 60, replace=False).astype(np.int32)
            new = rs.randint(-1, 4, size=60).astype(np.int32)
            same = rs.choice(np.setdiff1d(sids, ch), 40, replace=False).astype(np.int32)
            pool.set_stream_pool(np.concatenate([new, assign[same]]), np.concatenate([ch, same]))
            rep.rearm(ch[new != assign[ch]])
            assign[ch] = new
        if k == 7:
            cl = np.sort(rs.choice(S, 50, replace=False)).astype(np.int32)
            for x in banks + [pool]:
                x.clear(cuda(cl))
            rep.rearm(cl)
        if k in (10, 13):                        # reloads across activation classes: slot 1 (H = 12, Keras's defaults) takes
            slot, new = (1, 5) if k == 10 else (2, 3)    # model 5 (H = 24, tanh / sigmoid), slot 2 (tanh / sigmoid) model 3
            model, pr, sens, lvl = spec[new]
            assert spec[row[slot]][0].activation != model.activation and (assign == slot).any()
            pool.pool_load(slot, model, pr, sensitivity=sens, trigger_level=lvl)
            row[slot] = new
            rep.rearm(sids[assign == slot])
        c = cuda(noise(S, CHUNK, seed=300 + k))
        bo = run_banks(banks, c)
        po = pool.update_pool(c)
        mids = np.where(assign >= 0, row[np.maximum(assign, 0)], -1)
        _, conf, fired = check_tick(po, bo, sids, mids)
        rep.check(sids, mids, conf, fired)
    pool.set_pool(4)
    assert (pool.stream_pool() == -1).all()
    c = cuda(noise(S, CHUNK, seed=999))
    po = pool.update_pool(c)
    assert np.isnan(po['conf'].cpu().numpy()).all() and not po['fired'].cpu().numpy().any()
    torch.cuda.synchronize()
    for x in banks + [pool]:
        x.core.close()


@gpu
def test_pool_warp_tiles_only_equal_default_tiles():
    """pb_debug_pool_tiles(1) scores every position in warp tiles: outputs bit-identical to the default split into block and
    warp tiles, on full and partial ticks."""
    m = _mod()
    S = 700
    spec = pool_models(m)
    assign = assignment(S, len(spec), seed=41)
    a, b = pool_of(m, spec, S), pool_of(m, spec, S)
    for x in (a, b):
        x.set_stream_pool(assign)
    assert b.core.lib.pb_debug_pool_tiles(b.core._h, 1) == 0
    rs = np.random.RandomState(42)
    for k in range(8):
        sids = np.arange(S, dtype=np.int32) if k % 2 == 0 else np.sort(rs.choice(S, S // 2, replace=False)).astype(np.int32)
        c, ids = cuda(noise(sids.size, CHUNK, seed=600 + k)), (None if k % 2 == 0 else cuda(sids))
        oa, ob = a.update_pool(c, ids), b.update_pool(c, ids)
        for q in ('raw', 'conf', 'fired'):
            assert np.array_equal(oa[q].cpu().numpy().view(np.uint8), ob[q].cpu().numpy().view(np.uint8))
    assert int(a.pool_count.item()) == int(b.pool_count.item()) > 0
    for x in (a, b):
        x.core.close()


@gpu
def test_pool_errors_change_nothing():
    import torch
    m = _mod()
    from mycroft_precise_b200.core import PBError, make_config
    S = 32
    spec = pool_models(m)[:2]
    sb = m.StreamBatch(spec[0][0], S, chunk_samples=CHUNK)
    with pytest.raises(PBError):
        sb.set_stream_pool(np.zeros(S, np.int32))            # no pool yet
    with pytest.raises(PBError):
        sb.update_pool(torch.zeros((S, CHUNK), dtype=torch.int16, device='cuda'))
    with pytest.raises(ValueError):
        sb.set_pool(-1)
    with pytest.raises(ValueError):
        sb.set_pool(2 ** 24 + 1)
    sb.set_pool(3)
    sb.pool_load(0, spec[0][0], sensitivity=0.8, trigger_level=1)
    sb.pool_load(1, spec[1][0], spec[1][1])
    base = np.array([0, 1, -1] * 10 + [0, 0], np.int32)
    sb.set_stream_pool(base)
    bad = [
        (np.array([0, 1], np.int32), np.array([5, 5], np.int32)),     # duplicate stream id
        (np.array([0, 1], np.int32), np.array([5, S], np.int32)),     # stream id out of range
        (np.array([3, 0], np.int32), np.array([4, 5], np.int32)),     # model id out of range
        (np.array([1, -2], np.int32), np.array([4, 5], np.int32)),    # model id below -1
        (np.array([1, 2], np.int32), np.array([4, 5], np.int32)),     # slot 2 holds no model
    ]
    for models, ids in bad:
        with pytest.raises(ValueError):
            sb.set_stream_pool(models, ids)
        assert np.array_equal(sb.stream_pool(), base)
    with pytest.raises(ValueError):
        sb.pool_load(3, spec[0][0])                              # slot out of range
    with pytest.raises(NotImplementedError):
        sb.pool_load(2, m.GruModel.random(13, 32, seed=3))       # outside the fused family
    with pytest.raises(ValueError):
        sb.pool_load(2, m.GruModel.random(12, 20, seed=3), m.ListenerParams(n_mfcc=12))
    with pytest.raises(ValueError):
        sb.set_stream_pool(np.array([2], np.int32), np.array([0], np.int32))   # the failed loads left slot 2 empty
    # front-end fields through the C ABI (the Python layer refuses them before the call)
    lib = sb.core.lib
    model = spec[0][0]
    k, u, b, w = sb.core._weights(13, 20, model.kernel, model.recurrent, model.bias, model.dense_w)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    for field, value in (('hop_samples', 400), ('chunk_samples', 512), ('n_mfcc', 12), ('use_delta', 1)):
        cfg = make_config(sb.pr, 20, S, CHUNK)
        setattr(cfg, field, value)
        assert lib.pb_pool_load(sb.core._h, 2, C.byref(cfg), vp(k), vp(u), vp(b), vp(w), 0.0, None, 0) == -1
        assert field.encode() in lib.pb_last_error()
    cfg = make_config(sb.pr, 20, S, CHUNK)
    cd = np.zeros(7)
    assert lib.pb_pool_load(sb.core._h, 2, C.byref(cfg), vp(k), vp(u), vp(b), vp(w), 0.0, vp(cd), 7) == -1   # cd length
    assert np.array_equal(sb.stream_pool(), base)
    o = sb.update_pool(cuda(noise(S, CHUNK, seed=1)))
    assert np.isnan(o['conf'].cpu().numpy()[base < 0]).all() and not np.isnan(o['conf'].cpu().numpy()[base >= 0]).any()
    sb.set_pool(0)
    assert (sb.stream_pool() == -1).all()
    sb.core.close()


@gpu
def test_pool_two_cuda_streams():
    """Partial pool ticks over two halves of the streams, on two CUDA streams with no host synchronisation between them,
    equal the same ticks on one stream."""
    import torch
    m = _mod()
    S = 2000
    spec = pool_models(m)
    assign = assignment(S, len(spec), seed=12)
    a, b = pool_of(m, spec, S), pool_of(m, spec, S)
    a.set_stream_pool(assign)
    b.set_stream_pool(assign)
    perm = np.random.RandomState(13).permutation(S).astype(np.int32)
    halves = [cuda(np.sort(perm[:S // 2])), cuda(np.sort(perm[S // 2:]))]
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    for k in range(6):
        pcms = [cuda(noise(S // 2, CHUNK, seed=400 + 2 * k + h)) for h in range(2)]
        want = [a.update_pool(pcms[h], halves[h]) for h in range(2)]
        want = [{q: o[q].cpu().numpy() for q in o} for o in want]
        torch.cuda.synchronize()
        got = []
        for h, st in enumerate((s1, s2)):
            with torch.cuda.stream(st):
                got.append(b.update_pool(pcms[h], halves[h]))
        torch.cuda.synchronize()
        for h in range(2):
            for q in ('raw', 'conf', 'fired'):
                assert np.array_equal(bits(got[h][q].cpu().numpy()) if q != 'fired' else got[h][q].cpu().numpy(),
                                      bits(want[h][q]) if q != 'fired' else want[h][q])
    assert int(a.pool_count.item()) == int(b.pool_count.item()) > 0
    for x in (a, b):
        x.core.close()


@gpu
def test_pool_state_records():
    """Export / import between two pool handles continues bit-identically, refractory state included; the import sets the
    snapshot's pool models.  A handle without a pool writes 0 into pool_activation."""
    m = _mod()
    S = 500
    spec = pool_models(m)
    assign = assignment(S, len(spec), seed=21)
    a, b = pool_of(m, spec, S), pool_of(m, spec, S)
    a.set_stream_pool(assign)
    pcm = noise(S, 20 * CHUNK, seed=22)
    for k in range(10):
        a.update_pool(cuda(pcm[:, k * CHUNK:(k + 1) * CHUNK]))
    snap = a.export_streams()
    pa = snap['state'].cpu().numpy()[:, 56:60].copy().view(np.int32)[:, 0]
    assert (pa < 0).any() and (pa[assign < 0] == 0).all()
    assert np.array_equal(snap['stream_pool'], assign)
    b.import_streams(snap)
    assert np.array_equal(b.stream_pool(), assign)
    for k in range(10, 20):
        c = cuda(pcm[:, k * CHUNK:(k + 1) * CHUNK])
        oa, ob = a.update_pool(c), b.update_pool(c)
        for q in ('raw', 'conf'):
            assert np.array_equal(bits(oa[q].cpu().numpy()), bits(ob[q].cpu().numpy()))
        assert np.array_equal(oa['fired'].cpu().numpy(), ob['fired'].cpu().numpy())
    plain = m.StreamBatch(spec[0][0], S, chunk_samples=CHUNK)
    plain.update(cuda(pcm[:, :CHUNK]))
    rec = plain.export_streams()['state'].cpu().numpy()
    assert not rec[:, 56:64].any()
    # pool models a batch does not hold: refused before anything changes (masks included)
    small = pool_of(m, spec[:3], S)
    masked = dict(snap, stream_models=np.full(S, 0x01, np.uint8))
    for x in (plain, small):
        before = x.export_streams()
        with pytest.raises(ValueError, match='pool models'):
            x.import_streams(masked)
        after = x.export_streams()
        assert np.array_equal(before['state'].cpu().numpy(), after['state'].cpu().numpy())
        assert (x.core.stream_models() == 0xFF).all()
        assert ('stream_pool' in after) == (x is small) and (x.stream_pool() == -1).all()
    small.core.close()
    for x in (a, b, plain):
        x.core.close()


@gpu
def test_pool_history_and_clips():
    """History on pool ticks (uniform and ragged) returns the fed audio, and activation_audio takes the pool's [n] fired."""
    m = _mod()
    S, H = 64, 4000
    spec = pool_models(m)[:4]
    sb = pool_of(m, spec, S)
    assign = (np.arange(S) % 5 - 1).astype(np.int32)
    sb.set_stream_pool(assign)
    sb.set_history(samples=H)
    on = np.arange(S) % 3 != 0
    sb.set_stream_history(on)
    fed = [np.zeros(0, np.int16) for _ in range(S)]
    clips = 0
    rs = np.random.RandomState(31)
    for k in range(8):
        if k == 5:                                   # a ragged tick with odd offsets
            lens = rs.randint(1, 1500, size=S) | 1
            offs = np.concatenate([[1], 1 + np.cumsum(lens)]).astype(np.int64)
            flat = noise(1, int(offs[-1]), seed=500 + k)[0]
            o = sb.update_pool(cuda(flat), offsets=cuda(offs))
            for s in range(S):
                fed[s] = np.concatenate([fed[s], flat[offs[s]:offs[s + 1]]])
        else:
            pcm = noise(S, CHUNK, seed=500 + k)
            o = sb.update_pool(cuda(pcm))
            for s in range(S):
                fed[s] = np.concatenate([fed[s], pcm[s]])
        got = sb.read_history().cpu().numpy()
        for s in np.nonzero(on)[0]:
            tail = fed[s][-H:]
            assert np.array_equal(got[s, H - tail.size:], tail) and not got[s, :H - tail.size].any()
        act = sb.activation_audio(o['fired'])
        fired = np.nonzero(o['fired'].cpu().numpy())[0]
        assert sorted(act['stream'].cpu().numpy().tolist()) == [s for s in fired if on[s]]
        assert not act['slot'].cpu().numpy().any()
        for s, clip in zip(act['stream'].cpu().numpy(), act['audio'].cpu().numpy()):
            assert np.array_equal(clip, got[s])
        clips += len(act['stream'])
    assert clips > 0
    sb.core.close()


def test_pool_null_handle_is_invalid():
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
    out = np.zeros(4, np.int32)
    assert lib.pb_set_pool(None, 4) == -1 and b'null' in lib.pb_last_error()
    assert lib.pb_pool_load(None, 0, C.byref(cfg), p, p, p, p, 0.0, None, 0) == -1
    assert lib.pb_set_stream_pool(None, None, out.ctypes.data_as(C.c_void_p), 4) == -1
    assert lib.pb_get_stream_pool(None, None, 4, out.ctypes.data_as(C.c_void_p)) == -1
    assert lib.pb_update_pool(None, None, None, 0, None, 0, None, None, None, None, None) == -1
    assert lib.pb_debug_pool_tiles(None, 1) == -1
