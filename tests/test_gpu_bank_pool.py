"""Combined bank + pool ticks (pb_update_all) and per-stream pool trigger settings (pb_set_stream_pool_trigger).

The reference for every combined tick is a pair of twin handles fed the same audio: A holds the same bank (masks and
per-stream bank trigger settings included), B the same pool.  Rows 0 .. M-1 of the combined output must equal A's bank
tick bit for bit, row M B's pool tick.  Pool trigger settings are checked against OracleTrigger replayed over the GPU's own
conf.  -m gpu, except the null-handle check."""
import ctypes as C

import numpy as np
import pytest

from oracle.trigger import OracleTrigger

gpu = pytest.mark.gpu
CHUNK = 1024
CHUNK_BYTES = [1, 2048, 3000, 4096, 16385, 40000]       # refractory -16384, -8, -6, -4, -1, -1
LEVELS = [-1, 0, 1, 3, 10]


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
    """(model, params, sensitivity, trigger_level) of twelve fused networks with dense biases that make them fire."""
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
    return a.view({1: np.uint8, 4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


def host(o):
    return tuple(o[k].cpu().numpy() for k in ('raw', 'conf', 'fired'))


def bank_of(m, spec, S):
    """A batch whose bank is spec (slot i = spec[i])."""
    model, pr, sens, lvl = spec[0]
    sb = m.StreamBatch(model, S, params=pr, chunk_samples=CHUNK, sensitivity=sens, trigger_level=lvl)
    for model, pr, sens, lvl in spec[1:]:
        sb.add_model(model, pr, sensitivity=sens, trigger_level=lvl)
    return sb


def load_pool(sb, spec):
    sb.set_pool(len(spec))
    for i, (model, pr, sens, lvl) in enumerate(spec):
        sb.pool_load(i, model, pr, sensitivity=sens, trigger_level=lvl)
    return sb


def random_settings(rs, n, sens_choices):
    sens = np.asarray(sens_choices, np.float64)[rs.randint(0, len(sens_choices), n)]
    return sens, np.array(LEVELS, np.int32)[rs.randint(0, 5, n)], np.array(CHUNK_BYTES, np.int32)[rs.randint(0, 6, n)]


def tick_plan(rs, S, kinds):
    """(kind, sids, pcm, offsets, max_len) per tick: full, permuted, subset and ragged (odd offsets and lengths) ticks."""
    out = []
    for k, what in enumerate(kinds):
        if what == 'ragged':
            sids = rs.permutation(S)[:max(1, S - S // 7)].astype(np.int32)
            lens = rs.randint(1, 2 * CHUNK, size=sids.size)
            lens[::3] |= 1
            offs = np.concatenate([[3], 3 + np.cumsum(lens)]).astype(np.int64)
            out.append((what, sids, noise(1, int(offs[-1]), seed=rs.randint(1 << 30))[0], offs, int(lens.max())))
            continue
        if what == 'full':
            sids = np.arange(S, dtype=np.int32)
        elif what == 'perm':
            sids = rs.permutation(S).astype(np.int32)
        else:
            sids = np.sort(rs.choice(S, max(1, S // 3), replace=False)).astype(np.int32)
        out.append((what, sids, noise(sids.size, CHUNK, seed=rs.randint(1 << 30)), None, None))
    return out


def run_tick(sb, how, t):
    """One tick of plan entry t on sb: how = 'bank' (update_models / update_ragged), 'pool' (update_pool) or 'all'."""
    what, sids, pcm, offs, max_len = t
    ids = None if what == 'full' else cuda(sids)
    if offs is None:
        c = cuda(pcm)
        o = sb.update_models(c, ids) if how == 'bank' else getattr(sb, 'update_' + how)(c, ids)
    else:
        c, o_ = cuda(pcm), cuda(offs)
        if how == 'bank':
            o = sb.update_ragged(c, o_, ids, max_len)
        else:
            o = getattr(sb, 'update_' + how)(c, ids, offsets=o_, max_len=max_len)
    return host(o)


@gpu
@pytest.mark.parametrize('S', [300, 9000])
@pytest.mark.parametrize('M,routed,bank_trig', [(1, False, False), (1, True, True), (3, False, True), (3, True, False)])
def test_combined_tick_equals_twins(S, M, routed, bank_trig):
    m = _mod()
    spec = pool_models(m)
    bspec = spec[:M]
    assign = assignment(S, len(spec), seed=S + M)
    a = bank_of(m, bspec, S)                                     # A: the bank
    b = load_pool(m.StreamBatch(spec[0][0], S, chunk_samples=CHUNK), spec)    # B: the pool
    c = load_pool(bank_of(m, bspec, S), spec)                    # the combined handle
    for x in (b, c):
        x.set_stream_pool(assign)
    rs = np.random.RandomState(S * 10 + M)
    if routed:
        masks = rs.randint(0, 1 << M, size=S).astype(np.uint8)
        masks[:3] = 0                                            # some streams on no bank model
        for x in (a, c):
            x.set_stream_models(masks)
    if bank_trig:
        ids = rs.permutation(S)[:S * 2 // 3].astype(np.int32)
        sens, lvl, chunk = random_settings(rs, ids.size, (0.0, 1.0, 0.5, 0.3, 0.7))
        for x in (a, c):
            x.set_stream_trigger(M - 1, sens, lvl, chunk, ids=ids)
    for x in (a, c):
        x.core.profile(True)
    kinds = ['full', 'perm', 'subset', 'ragged', 'full', 'subset', 'ragged', 'perm', 'full', 'ragged', 'full']
    fires = np.zeros(M + 1, np.int64)
    for t in tick_plan(rs, S, kinds):
        oa, ob, oc = run_tick(a, 'bank', t), run_tick(b, 'pool', t), run_tick(c, 'all', t)
        for q in range(3):
            assert oc[q].shape == (M + 1, t[1].size)
            assert np.array_equal(bits(oc[q][:M]), bits(oa[q].reshape(M, -1))), (t[0], q)
            assert np.array_equal(bits(oc[q][M]), bits(ob[q])), (t[0], q)
        assert np.array_equal(c.counts.cpu().numpy(), a.counts.cpu().numpy())
        assert int(c.pool_count.item()) == int(b.pool_count.item())
        fires += oc[2].sum(axis=1).astype(np.int64)
    print('S = %d, M = %d: fires per row %s' % (S, M, fires.tolist()))
    assert fires[M] > 0 and fires[:M].sum() > 0
    ra, rb, rc = (x.export_streams()['state'].cpu().numpy() for x in (a, b, c))
    assert np.array_equal(rc[:, :56], ra[:, :56]) and np.array_equal(rc[:, 60:], ra[:, 60:])
    assert np.array_equal(rc[:, 56:60], rb[:, 56:60])
    assert (rb[:, 56:60].view(np.int32) != 0).any()
    (_, la), (_, lc) = a.core.profile_read(), c.core.profile_read()
    assert la[0] == lc[0] > 0, (la, lc)                          # K1 runs once per combined tick
    for x in (a, b, c):
        x.core.close()


@gpu
def test_combined_history_appended_once_and_clips():
    """History after combined ticks (uniform and ragged) is exactly the fed audio, and activation_audio on the [M + 1, n]
    output returns the clips of pool fires as slot M."""
    m = _mod()
    S, H, M = 64, 6000, 2
    spec = pool_models(m)
    sb = load_pool(bank_of(m, spec[:M], S), spec[:5])
    assign = (np.arange(S) % 6 - 1).astype(np.int32)
    sb.set_stream_pool(assign)
    sb.set_history(samples=H)
    on = np.arange(S) % 3 != 0
    sb.set_stream_history(on)
    fed = [np.zeros(0, np.int16) for _ in range(S)]
    clips = np.zeros(M + 1, np.int64)
    rs = np.random.RandomState(31)
    for k in range(9):
        if k in (3, 6):
            lens = rs.randint(1, 1500, size=S) | 1
            offs = np.concatenate([[1], 1 + np.cumsum(lens)]).astype(np.int64)
            flat = noise(1, int(offs[-1]), seed=500 + k)[0]
            o = sb.update_all(cuda(flat), offsets=cuda(offs))
            for s in range(S):
                fed[s] = np.concatenate([fed[s], flat[offs[s]:offs[s + 1]]])
        else:
            pcm = noise(S, CHUNK, seed=500 + k)
            o = sb.update_all(cuda(pcm))
            for s in range(S):
                fed[s] = np.concatenate([fed[s], pcm[s]])
        got = sb.read_history().cpu().numpy()
        for s in np.nonzero(on)[0]:
            tail = fed[s][-H:]
            assert np.array_equal(got[s, H - tail.size:], tail) and not got[s, :H - tail.size].any(), (k, s)
        act = sb.activation_audio(o['fired'])
        f = o['fired'].cpu().numpy()
        want = sorted((int(r), int(s)) for r, s in zip(*np.nonzero(f)) if on[s])
        assert sorted(zip(act['slot'].cpu().numpy().tolist(), act['stream'].cpu().numpy().tolist())) == want
        for slot, s, clip in zip(act['slot'].cpu().numpy(), act['stream'].cpu().numpy(), act['audio'].cpu().numpy()):
            assert np.array_equal(clip, got[s])
            clips[slot] += 1
    print('clips per row', clips.tolist())
    assert clips[M] > 0
    sb.core.close()


@gpu
def test_combined_refused_calls_change_nothing():
    import torch
    m = _mod()
    from mycroft_precise_b200.core import PBError
    S = 40
    spec = pool_models(m)
    a, b = bank_of(m, spec[:2], S), bank_of(m, spec[:2], S)
    pcm0 = cuda(noise(S, CHUNK, seed=1))
    with pytest.raises(PBError, match='pool'):
        a.update_all(pcm0)                                       # no pool
    for x in (a, b):
        load_pool(x, spec[:3])
        x.set_stream_pool((np.arange(S) % 4 - 1).astype(np.int32))
    for x in (a, b):
        x.update_all(pcm0)
    lib, h = a.core.lib, a.core._h
    conf = torch.empty((3, S), dtype=torch.float64, device='cuda')
    offs = cuda(np.arange(S + 1, dtype=np.int64) * 100)
    flat = cuda(noise(1, 100 * S, seed=2)[0])
    vp = lambda t: C.c_void_p(t.data_ptr())
    calls = [
        (-1, (vp(pcm0), None, 0, None, S, None, None, None, None, None, None)),                 # null d_conf
        (-1, (vp(pcm0), None, 0, None, S + 1, None, vp(conf), None, None, None, None)),         # n > max_streams
        (-1, (vp(pcm0), None, 0, None, -1, None, vp(conf), None, None, None, None)),            # n < 0
        (-1, (None, None, 0, None, S, None, vp(conf), None, None, None, None)),                 # null pcm
        (-1, (vp(flat), vp(offs), 0, None, S, None, vp(conf), None, None, None, None)),         # max_len < 1
    ]
    for rc, args in calls:
        assert lib.pb_update_all(h, *args) == rc, lib.pb_last_error()
    assert lib.pb_debug_k1_mode(h, 2) == 0
    assert lib.pb_update_all(h, vp(flat), vp(offs), 100, None, S, None, vp(conf), None, None, None, None) == -4
    assert b'k1 mode' in lib.pb_last_error()
    assert lib.pb_debug_k1_mode(h, 0) == 0
    with pytest.raises(ValueError):
        a.update_all(flat, offsets=offs, max_len=0)
    with pytest.raises(ValueError):
        a.update_all(cuda(noise(S, CHUNK - 1, seed=3)))
    # a pool on a handle without slot-0 weights
    bare = m.PreciseB200(max_streams=S, chunk_samples=CHUNK)
    bare.set_pool(1)
    with pytest.raises(PBError, match='pb_load_weights'):
        bare.update_all(pcm0)
    bare.close()
    torch.cuda.synchronize()
    assert np.array_equal(a.export_streams()['state'].cpu().numpy(), b.export_streams()['state'].cpu().numpy())
    for k in range(3):
        c = cuda(noise(S, CHUNK, seed=10 + k))
        oa, ob = host(a.update_all(c)), host(b.update_all(c))
        for q in range(3):
            assert np.array_equal(bits(oa[q]), bits(ob[q]))
    assert np.array_equal(a.export_streams()['state'].cpu().numpy(), b.export_streams()['state'].cpu().numpy())
    assert np.array_equal(a.counts.cpu().numpy(), b.counts.cpu().numpy()) and int(a.pool_count) == int(b.pool_count)
    for x in (a, b):
        x.core.close()


class PoolReplay:
    """OracleTrigger per stream over the pool row: the stream's own settings, or its model's while it follows the model;
    fresh on an arm, a changed setting, a changed model, a clear and a reload of its model."""

    def __init__(self, spec, S):
        self.spec, self.det, self.own = spec, [None] * S, [None] * S
        self.fired = 0
        self.events = {}

    def rearm(self, sids):
        for s in np.atleast_1d(sids):
            self.det[int(s)] = None

    def set(self, sids, sens, lvl, chunk):
        n = len(sids)
        for s, x, l, c in zip(sids, np.broadcast_to(sens, n), np.broadcast_to(lvl, n), np.broadcast_to(chunk, n)):
            new = None if int(c) == 0 else (int(c), np.float64(x).tobytes(), int(l))
            if new != self.own[int(s)]:
                self.det[int(s)] = None
            self.own[int(s)] = new

    def check(self, sids, mids, conf, fired):
        want = np.zeros(len(sids), np.uint8)
        for j, (s, mid) in enumerate(zip(sids, mids)):
            if mid < 0:
                continue
            d = self.det[s]
            if d is None:
                own = self.own[s]
                if own is None:
                    _, _, sens, lvl = self.spec[mid]
                    d = OracleTrigger(2 * CHUNK, sens, lvl)
                else:
                    d = OracleTrigger(own[0], float(np.frombuffer(own[1], np.float64)[0]), own[2])
                d.n_fired = 0
                self.det[s] = d
            want[j] = d.update(float(conf[j]))
            if want[j]:
                d.n_fired += 1
                ev = self.events.setdefault(d.chunk_size, [0, 0])
                ev[0] += d.n_fired == 1
                ev[1] += d.n_fired == 2
        bad = np.nonzero(fired != want)[0]
        assert bad.size == 0, 'fired differs from the oracle at %d items, first stream %d' % (bad.size, sids[bad[0]])
        self.fired += int(want.sum())


def n_fires(confs, chunk, sens, lvl):
    d = OracleTrigger(chunk, sens, lvl)
    return sum(d.update(float(c)) for c in confs)


@gpu
@pytest.mark.parametrize('S', [7, 9000])
def test_pool_trigger_settings_follow_oracle(S):
    """Random (sensitivity, level, chunk_bytes) per stream, some streams following their model, through update_pool and
    through update_all.  Six streams, one per chunk size, get level -1 and a sensitivity chosen from their own conf so that
    each fires, and fires again after its refractory period (chunk 1 fires once); some streams sit exactly on a tie."""
    m = _mod()
    spec = pool_models(m)
    rs = np.random.RandomState(S)
    assign = np.array([0, 1, 2, 3, 4, 5, -1], np.int32) if S == 7 else assignment(S, len(spec), seed=S)
    twin = load_pool(m.StreamBatch(spec[0][0], S, chunk_samples=CHUNK), spec)
    p = load_pool(m.StreamBatch(spec[0][0], S, chunk_samples=CHUNK), spec)
    c = load_pool(bank_of(m, spec[:2], S), spec)
    for x in (twin, p, c):
        x.set_stream_pool(assign)
    ticks = tick_plan(rs, S, ['full', 'perm', 'subset'] * 10)
    ot =[run_tick(twin, 'pool', t) for t in ticks]               # the twin first: its conf chooses the settings
    conf_all = np.concatenate([o[1][~np.isnan(o[1])] for o in ot])
    sens_choices = np.r_[0.0, 1.0, 0.5, 1.0 - np.quantile(conf_all, [0.3, 0.6, 0.9])]
    sens, lvl, chunk = random_settings(rs, S, sens_choices)
    chunk[rs.rand(S) < 0.15] = 0                                 # these follow their model
    on = np.nonzero(assign >= 0)[0]
    perm = rs.permutation(on).astype(np.int32)
    for ci, sid in enumerate(perm[:6]):
        hist = [o[1][list(t[1]).index(sid)] for t, o in zip(ticks, ot) if sid in t[1]]
        need = 1 if CHUNK_BYTES[ci] == 1 else 2
        cands = [1.0 - np.quantile(hist, q) for q in np.linspace(0.5, 0.97, 16)]
        ok = [x for x in cands if n_fires(hist, CHUNK_BYTES[ci], x, -1) >= need]
        assert ok, 'no sensitivity makes stream %d fire %d times over %s' % (sid, need, hist)
        chunk[sid], lvl[sid], sens[sid] = CHUNK_BYTES[ci], -1, ok[0]
    ties = perm[6:6 + max(0, on.size // 20)]
    for sid in ties:                                             # 1 - sens == an observed conf >= 0.5 exactly
        hist = np.array([o[1][list(t[1]).index(sid)] for t, o in zip(ticks, ot) if sid in t[1]])
        big = hist[hist >= 0.5]
        if big.size:
            sens[sid], lvl[sid], chunk[sid] = 1.0 - big[0], 0, 2048
    for x in (p, c):
        half = rs.permutation(S).astype(np.int32)
        for ids in (half[:S // 2], half[S // 2:]):
            x.set_stream_pool_trigger(sens[ids], lvl[ids], chunk[ids], ids=ids)
    got = p.stream_pool_trigger()
    follow = chunk == 0
    assert np.isnan(got[0][follow]).all() and not got[1][follow].any() and not got[2][follow].any()
    assert np.array_equal(bits(got[0][~follow]), bits(sens[~follow]))
    assert np.array_equal(got[1][~follow], lvl[~follow]) and np.array_equal(got[2][~follow], chunk[~follow])
    for x in (c.stream_pool_trigger(),):
        for q in range(3):
            assert np.array_equal(bits(x[q]), bits(got[q]))
    reps = [PoolReplay(spec, S), PoolReplay(spec, S)]
    for r in reps:
        r.set(np.arange(S), sens, lvl, chunk)
    n_ties = 0
    for t, o in zip(ticks, ot):
        sids = t[1]
        op, oc = run_tick(p, 'pool', t), run_tick(c, 'all', t)
        for q in range(2):
            assert np.array_equal(bits(op[q]), bits(o[q])) and np.array_equal(bits(oc[q][2]), bits(o[q]))
        reps[0].check(sids, assign[sids], op[1], op[2])
        reps[1].check(sids, assign[sids], oc[1][2], oc[2][2])
        n_ties += int((op[1] == 1.0 - sens[sids])[np.isin(sids, ties)].sum())
    print('events per chunk size', reps[0].events, 'fired', reps[0].fired, 'ties', n_ties)
    for cb in CHUNK_BYTES:
        ev = reps[0].events.get(cb, [0, 0])
        assert ev[0] >= 1 and (cb == 1 or ev[1] >= 1), (cb, ev)
    if S > 7:
        assert n_ties >= 1
    assert int(p.pool_count.item()) == reps[0].fired and int(c.pool_count.item()) == reps[1].fired
    for x in (twin, p, c):
        x.core.close()


@gpu
def test_pool_trigger_model_values_equal_unset():
    """Every stream set to its model's own (sensitivity, level, 2 * chunk_samples) before the first tick, and set to the same
    values again after ticks ran (unchanged: the detectors keep their state), through update_pool and update_all: fired and
    counts equal the untouched twin's tick for tick.  chunk_bytes 0 on a set stream reads back as (NaN, 0, 0)."""
    m = _mod()
    S = 2000
    spec = pool_models(m)
    assign = assignment(S, len(spec), seed=3)
    rs = np.random.RandomState(4)
    mods = np.maximum(assign, 0)
    sens = np.array([x[2] for x in spec])[mods]
    lvl = np.array([x[3] for x in spec], np.int32)[mods]
    for how in ('pool', 'all'):
        a = load_pool(bank_of(m, spec[:1], S), spec)
        b = load_pool(bank_of(m, spec[:1], S), spec)
        for x in (a, b):
            x.set_stream_pool(assign)
        for k, t in enumerate(tick_plan(rs, S, ['full', 'perm', 'subset', 'ragged'] * 2)):
            if k == 0:
                for r in (0, 1):
                    a.set_stream_pool_trigger(sens[r::2], lvl[r::2], 2 * CHUNK, ids=np.arange(r, S, 2, dtype=np.int32))
            if k == 3:
                a.set_stream_pool_trigger(sens, lvl, 2 * CHUNK)
            oa, ob = run_tick(a, how, t), run_tick(b, how, t)
            for q in range(3):
                assert np.array_equal(bits(oa[q]), bits(ob[q])), (how, k, q)
        assert int(a.pool_count.item()) == int(b.pool_count.item()) > 0
        a.set_stream_pool_trigger(0.3, 1, 0, ids=np.array([5, 6], np.int32))
        s, l, cb = a.stream_pool_trigger(np.array([5, 6, 7], np.int32))
        assert np.isnan(s[:2]).all() and not l[:2].any() and not cb[:2].any() and cb[2] == 2 * CHUNK
        for x in (a, b):
            x.core.close()


@gpu
def test_pool_trigger_rules():
    """Re-arm and keep: a changed entry re-arms, an unchanged one keeps the detector; chunk_bytes 0 returns a stream to its
    model's values; settings survive set_stream_pool (a changed model re-arms), pool_load (re-arms its streams) and clear
    (re-arms); set_pool drops them."""
    m = _mod()
    S = 400
    spec = pool_models(m)[:6]
    sb = load_pool(bank_of(m, spec[:1], S), spec[:4])
    rs = np.random.RandomState(9)
    assign = rs.randint(-1, 4, size=S).astype(np.int32)
    sb.set_stream_pool(assign)
    pspec = list(spec[:4])
    rep = PoolReplay(pspec, S)
    sens, lvl, chunk = random_settings(rs, S, (0.0, 0.3, 0.5, 0.8, 1.0))
    sids = np.arange(S, dtype=np.int32)
    for k in range(18):
        if k == 0:
            sb.set_stream_pool_trigger(sens, lvl, chunk)
            rep.set(sids, sens, lvl, chunk)
        if k == 3:                               # some entries change, others are set to what they are
            ch = rs.choice(S, 80, replace=False).astype(np.int32)
            sens[ch[:40]] = np.where(sens[ch[:40]] == 0.5, 0.8, 0.5)
            chunk[ch[40:60]] = 0                 # back to the model
            sb.set_stream_pool_trigger(sens[ch], lvl[ch], chunk[ch], ids=ch)
            rep.set(ch, sens[ch], lvl[ch], chunk[ch])
        if k == 5:                               # model changes re-arm, settings stay
            ch = rs.choice(S, 60, replace=False).astype(np.int32)
            new = rs.randint(-1, 4, size=60).astype(np.int32)
            sb.set_stream_pool(new, ch)
            rep.rearm(ch[new != assign[ch]])
            assign[ch] = new
        if k == 8:
            cl = np.sort(rs.choice(S, 50, replace=False)).astype(np.int32)
            sb.clear(cuda(cl))
            rep.rearm(cl)
        if k == 11:                              # a reload re-arms the slot's streams and keeps their settings
            model, pr, s_, l_ = spec[5]
            sb.pool_load(1, model, pr, sensitivity=s_, trigger_level=l_)
            pspec[1] = spec[5]
            rep.rearm(sids[assign == 1])
        got = sb.stream_pool_trigger()
        own = chunk != 0
        assert np.array_equal(bits(got[0][own]), bits(sens[own])) and np.array_equal(got[2][own], chunk[own])
        assert np.isnan(got[0][~own]).all() and not got[2][~own].any()
        o = host(sb.update_all(cuda(noise(S, CHUNK, seed=300 + k))) if k % 2 else sb.update_pool(cuda(noise(S, CHUNK, seed=300 + k))))
        conf, fired = (o[1][1], o[2][1]) if k % 2 else (o[1], o[2])
        rep.check(sids, assign, conf, fired)
    assert rep.fired > 0
    sb.set_pool(4)                               # replaced: every stream on none, settings dropped
    s, l, cb = sb.stream_pool_trigger()
    assert np.isnan(s).all() and not l.any() and not cb.any()
    sb.set_pool(0)
    s, l, cb = sb.stream_pool_trigger()
    assert np.isnan(s).all() and not l.any() and not cb.any()
    sb.core.close()


@gpu
def test_pool_trigger_snapshot_and_validation():
    """A snapshot carries the pool trigger settings into a second batch, which then continues bit-identically; malformed
    entries and refused setter calls change nothing."""
    m = _mod()
    from mycroft_precise_b200.core import PBError
    S = 500
    spec = pool_models(m)
    assign = assignment(S, len(spec), seed=21)
    a, b = (load_pool(bank_of(m, spec[:2], S), spec) for _ in range(2))
    a.set_stream_pool(assign)
    rs = np.random.RandomState(22)
    sens, lvl, chunk = random_settings(rs, S, (0.0, 0.3, 0.5, 0.8))
    chunk[::7] = 0
    a.set_stream_pool_trigger(sens, lvl, chunk)
    pcm = noise(S, 16 * CHUNK, seed=23)
    for k in range(8):
        a.update_all(cuda(pcm[:, k * CHUNK:(k + 1) * CHUNK]))
    snap = a.export_streams()
    assert 'stream_pool_trigger' in snap
    before = b.export_streams()
    for bad in ((sens, lvl), (sens[:-1], lvl, chunk), (sens, lvl, chunk.astype(np.float64)), (sens, lvl, np.where(chunk == 0, -1, chunk))):
        with pytest.raises(ValueError):
            b.import_streams(dict(snap, stream_pool_trigger=bad))
        after = b.export_streams()
        assert np.array_equal(before['state'].cpu().numpy(), after['state'].cpu().numpy())
        assert (b.stream_pool() == -1).all() and np.isnan(b.stream_pool_trigger()[0]).all()
    b.import_streams(snap)
    for q in range(3):
        assert np.array_equal(bits(b.stream_pool_trigger()[q]), bits(a.stream_pool_trigger()[q]))
    for k in range(8, 16):
        c = cuda(pcm[:, k * CHUNK:(k + 1) * CHUNK])
        oa, ob = host(a.update_all(c)), host(b.update_all(c))
        for q in range(3):
            assert np.array_equal(bits(oa[q]), bits(ob[q]))
    # the setter validates everything first
    cur = a.stream_pool_trigger()
    bad = [
        dict(ids=np.array([3, 3], np.int32)), dict(ids=np.array([3, S], np.int32)), dict(ids=np.array([-1, 3], np.int32)),
        dict(ids=np.array([3, 4], np.int32), chunk=-1),
    ]
    for case in bad:
        with pytest.raises(ValueError):
            a.set_stream_pool_trigger(0.9, 1, case.get('chunk', 2048), ids=case['ids'])
    lib = a.core.lib
    ids = np.array([3, 4], np.int32)
    s, l, cb = np.full(2, 0.9), np.full(2, 1, np.int32), np.array([2048, -1], np.int32)
    vp = lambda x: x.ctypes.data_as(C.c_void_p)
    assert lib.pb_set_stream_pool_trigger(a.core._h, vp(ids), vp(s), vp(l), vp(cb), 2) == -1
    for q in range(3):
        assert np.array_equal(bits(a.stream_pool_trigger()[q]), bits(cur[q]))
    plain = bank_of(m, spec[:1], 8)
    with pytest.raises(PBError, match='pool'):
        plain.set_stream_pool_trigger(0.5, 3, 2048)
    s, l, cb = plain.stream_pool_trigger()
    assert np.isnan(s).all() and not l.any() and not cb.any()
    with pytest.raises(ValueError):
        plain.set_stream_pool_trigger(np.array(['a']), 3, 2048)
    for x in (a, b, plain):
        x.core.close()


def test_bank_pool_null_handle_is_invalid():
    import os
    import __graft_entry__ as g
    from mycroft_precise_b200.core import lib_path, get_lib
    if not os.path.isfile(lib_path()):
        g.build()
    lib = get_lib()
    d = np.zeros(4, np.float64)
    i = np.zeros(4, np.int32)
    pd, pi = d.ctypes.data_as(C.c_void_p), i.ctypes.data_as(C.c_void_p)
    assert lib.pb_update_all(None, None, None, 0, None, 0, None, None, None, None, None, None) == -1
    assert b'null' in lib.pb_last_error()
    assert lib.pb_set_stream_pool_trigger(None, None, pd, pi, pi, 4) == -1
    assert lib.pb_get_stream_pool_trigger(None, None, 4, pd, pi, pi) == -1
    assert lib.pb_set_stream_pool_trigger(None, None, None, None, None, 0) == -1
