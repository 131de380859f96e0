"""Per-stream TriggerDetector settings (pb_set_stream_trigger): every tick entry point, the state rules and the API.

-m gpu, except the C-ABI null-handle check at the end.  A handle with settings must return raw and conf bit-identical to an
identical handle without them, and fired / counts equal to OracleTrigger(chunk_bytes, sensitivity, trigger_level) per
(stream, model), built when the detector is (re-)armed and replayed over the conf the GPU returned.
"""
import ctypes as C

import numpy as np
import pytest

from oracle.trigger import OracleTrigger
from test_gpu_model_bank import bank_models
from test_gpu_stream_models import bank, cuda, host, noise

gpu = pytest.mark.gpu
CHUNK = 1024
CHUNK_BYTES = [1, 2048, 3000, 4096, 16385, 40000]       # refractory -16384, -8, -6, -4, -1, -1
LEVELS = [-1, 0, 1, 3, 10]


def _mod():
    import mycroft_precise_b200 as m
    return m


def hot_model(m, seed=8):
    model = m.GruModel.random(13, 20, seed=seed, scale=0.1)
    model.dense_b = 3.0                                                # confidences often high
    return model


def key(setting):
    """A setting compared as the library compares it: the sensitivity bit for bit."""
    c, s, lvl = setting
    return int(c), np.float64(s).tobytes(), int(lvl)


class Replay:
    """The oracle side of a handle with settings: one OracleTrigger per (stream, model), built with the stream's settings when
    the pair is first scored after an arm, a clear, a changed setting or a subscription bit going from 0 to 1."""

    def __init__(self, spec):
        self.default = [(2 * CHUNK, float(sens), int(lvl)) for _, _, sens, lvl in spec]
        self.settings = {}
        self.det = {}
        self.fired = np.zeros(len(spec), np.int64)
        self.events = {}                     # chunk_bytes -> [detectors that fired, detectors that fired a second time]

    def setting(self, sid, mi):
        return self.settings.get((sid, mi), self.default[mi] if mi < len(self.default) else None)

    def set(self, mi, sids, sens, lvl, chunk):
        n = len(sids)
        for sid, s, l, c in zip(sids, np.broadcast_to(sens, n), np.broadcast_to(lvl, n), np.broadcast_to(chunk, n)):
            new = (int(c), float(s), int(l))
            if key(new) != key(self.setting(int(sid), mi)):
                self.det.pop((int(sid), mi), None)
            self.settings[(int(sid), mi)] = new

    def clear(self, sids):
        for sid in sids:
            for mi in range(8):
                self.det.pop((int(sid), mi), None)

    def set_masks(self, old, new, sids):
        for sid in sids:
            for mi in range(8):
                if (new[sid] >> mi) & 1 and not (old[sid] >> mi) & 1:
                    self.det.pop((int(sid), mi), None)

    def tick(self, sids, a, b=None, mask=None):
        """a = (raw, conf, fired) of the handle with settings, b = (raw, conf) of its twin without, each [M, n] or [n]."""
        ra, ca, fa = (np.asarray(x).reshape(-1, len(sids)) for x in a)
        M = ra.shape[0]
        if mask is None:
            sub = np.ones((M, len(sids)), bool)
        else:
            sub = ((mask[sids][None, :] >> np.arange(M)[:, None]) & 1).astype(bool)
        if b is not None:
            rb, cb = (np.asarray(x).reshape(M, -1) for x in b)
            assert np.array_equal(ra[sub].view(np.uint32), rb[sub].view(np.uint32)), 'raw differs from the twin'
            assert np.array_equal(ca[sub].view(np.uint64), cb[sub].view(np.uint64)), 'conf differs from the twin'
        assert np.isnan(ra[~sub]).all() and np.isnan(ca[~sub]).all() and not fa[~sub].any()
        want = np.zeros_like(fa, dtype=bool)
        for mi, j in zip(*np.nonzero(sub)):
            k = (int(sids[j]), int(mi))
            d = self.det.get(k)
            if d is None:
                d = self.det[k] = OracleTrigger(*self.setting(*k))
                d.n_fired = 0
            want[mi, j] = d.update(float(ca[mi, j]))
            if want[mi, j]:
                d.n_fired += 1
                ev = self.events.setdefault(d.chunk_size, [0, 0])
                ev[0] += d.n_fired == 1
                ev[1] += d.n_fired == 2
        bad = np.nonzero(fa.astype(bool) != want)
        assert bad[0].size == 0, 'fired differs from the oracle at %d pairs, first (model, stream) %s, setting %s' % (
            bad[0].size, (int(bad[0][0]), int(sids[bad[1][0]])), self.setting(int(sids[bad[1][0]]), int(bad[0][0])))
        self.fired[:M] += fa.sum(axis=1).astype(np.int64)
        return sub


def plan(rs, S, K):
    """K ticks: full, permuted and partial (half) id sets in turn, with seeded PCM."""
    out = []
    for k in range(K):
        kind = k % 3
        sids = np.arange(S, dtype=np.int32) if kind == 0 else rs.permutation(S)[:S if kind == 1 else S // 2 + 1].astype(np.int32)
        out.append((sids, noise((len(sids), CHUNK), rs)))
    return out


def run(sb, ticks):
    return [host(sb.update(cuda(pcm), cuda(sids))) for sids, pcm in ticks]


def n_fires(confs, chunk, sens, lvl):
    d = OracleTrigger(chunk, sens, lvl)
    return sum(d.update(float(c)) for c in confs)


@gpu
@pytest.mark.parametrize('S', [7, 9000])
def test_one_model_settings_follow_oracle(S):
    """Random (sensitivity, level, chunk_bytes) per stream on a one-model handle: the warp kernel (partial ticks, and S = 7) and
    the bank-kernel scan (9 000 streams).  Six streams, one per chunk size, get level -1 and a sensitivity picked from their
    own conf history so that each fires, and fires again after its refractory period (chunk 1, refractory -16 384, fires)."""
    m = _mod()
    rs = np.random.RandomState(S)
    spec = [(hot_model(m), None, 0.5, 3)]
    a, b = bank(m, spec, S), bank(m, spec, S)
    ticks = plan(rs, S, 30)
    ob = run(b, ticks)                                                 # the twin first: its conf chooses the settings
    conf_all = np.concatenate([o[1] for o in ob])
    sens_choices = np.r_[0.0, 1.0, 0.5, 1.0 - np.quantile(conf_all, [0.3, 0.6, 0.9])]
    chunk = np.array(CHUNK_BYTES, np.int32)[rs.randint(0, 6, S)]
    lvl = np.array(LEVELS, np.int32)[rs.randint(0, 5, S)]
    sens = sens_choices[rs.randint(0, len(sens_choices), S)]
    perm = rs.permutation(S).astype(np.int32)
    for ci, sid in enumerate(perm[:6]):
        hist = [o[1][list(sids).index(sid)] for (sids, _), o in zip(ticks, ob) if sid in sids]
        need = 1 if CHUNK_BYTES[ci] == 1 else 2
        cands = [1.0 - np.quantile(hist, q) for q in np.linspace(0.5, 0.97, 16)]
        ok = [s for s in cands if n_fires(hist, CHUNK_BYTES[ci], s, -1) >= need]
        assert ok, 'no sensitivity makes stream %d fire %d times over %s' % (sid, need, hist)
        chunk[sid], lvl[sid], sens[sid] = CHUNK_BYTES[ci], -1, ok[0]
    h1, h2 = S // 2, S - max(1, S // 10)                               # streams perm[h2:] keep the defaults
    for ids in (perm[:h1], perm[h1:h2]):
        a.set_stream_trigger(0, sens[ids], lvl[ids], chunk[ids], ids=ids)
    got = a.stream_trigger(0, perm)
    assert np.array_equal(got[0][:h2].view(np.uint64), sens[perm[:h2]].view(np.uint64))
    assert np.array_equal(got[1][:h2], lvl[perm[:h2]]) and np.array_equal(got[2][:h2], chunk[perm[:h2]])
    assert np.all(got[0][h2:] == 0.5) and np.all(got[1][h2:] == 3) and np.all(got[2][h2:] == 2048)
    rep = Replay(spec)
    rep.set(0, perm[:h2], sens[perm[:h2]], lvl[perm[:h2]], chunk[perm[:h2]])
    for (sids, pcm), o in zip(ticks, ob):
        rep.tick(sids, host(a.update(cuda(pcm), cuda(sids))), o[:2])
    print('events per chunk size', rep.events, 'fired', rep.fired)
    for c in CHUNK_BYTES:
        ev = rep.events.get(c, [0, 0])
        assert ev[0] >= 1 and (c == 1 or ev[1] >= 1), (c, ev)
    assert int(a.count.item()) == rep.fired[0]
    for x in (a, b):
        x.core.close()


class GeTrigger(OracleTrigger):
    """The debouncer with `>=` in place of `>`: what a tie would do if it counted as hot."""

    def update(self, prob):
        return OracleTrigger.update(self, np.nextafter(prob, 2.0))


@gpu
def test_tie_is_not_hot():
    """sensitivity = 1.0 - c for observed conf values c >= 0.5: 1.0 - sensitivity == c exactly (Sterbenz), and a tick whose conf
    equals the threshold is not hot."""
    m = _mod()
    S, K = 64, 12
    rs = np.random.RandomState(1)
    model = hot_model(m, seed=4)
    model.dense_b = 5.0                                                # confidences mostly above 0.5
    spec = [(model, None, 0.5, 3)]
    a, b = bank(m, spec, S), bank(m, spec, S)
    ticks = [(np.arange(S, dtype=np.int32), noise((S, CHUNK), rs)) for _ in range(K)]
    ob = run(b, ticks)
    conf = np.stack([o[1] for o in ob])                                # [K, S]
    c = np.array([rs.choice(col[col >= 0.5]) if (col >= 0.5).any() else col.max() for col in conf.T])
    big = c >= 0.5
    assert big.sum() >= S // 2, c
    sens = 1.0 - c
    assert np.array_equal((1.0 - sens[big]).view(np.uint64), c[big].view(np.uint64))
    a.set_stream_trigger(0, sens, 0, 2048)
    rep = Replay(spec)
    rep.set(0, np.arange(S), sens, 0, 2048)
    fired = []
    for (sids, pcm), o in zip(ticks, ob):
        oa = host(a.update(cuda(pcm)))
        rep.tick(sids, oa, o[:2])
        fired.append(oa[2].astype(bool))
    fired = np.stack(fired)
    differs = 0
    for s in np.nonzero(big)[0]:
        g = GeTrigger(2048, sens[s], 0)
        differs += [g.update(conf[k, s]) for k in range(K)] != list(fired[:, s])
    ties = int((conf[:, big] == (1.0 - sens[big])[None, :]).sum())
    print('ties', ties, 'streams where >= would differ', differs)
    assert ties >= big.sum() and differs > 0
    for x in (a, b):
        x.core.close()


@gpu
def test_settings_equal_to_defaults_change_nothing():
    """Every stream set to its model's own values, on a one-model handle (warp and bank-kernel paths) and on the four-model
    bank, some of them after ticks have run: fired and counts equal the untouched twin's tick for tick."""
    m = _mod()
    rs = np.random.RandomState(7)
    for spec, S, tick in (([(hot_model(m), None, 0.5, 3)], 9000, 'update'), (bank_models(m), 2000, 'update_models')):
        a, b = bank(m, spec, S), bank(m, spec, S)
        for k in range(8):
            for mi, (_, _, sens, lvl) in enumerate(spec):
                if (k == 0 and mi % 2 == 0) or k == 3:                 # at k = 3 the even slots are set a second time
                    a.set_stream_trigger(mi, sens, lvl, 2 * CHUNK)
            sids = np.arange(S, dtype=np.int32) if k % 2 == 0 else rs.permutation(S)[:S // 2].astype(np.int32)
            c, ids = cuda(noise((len(sids), CHUNK), rs)), cuda(sids)
            oa, ob = host(getattr(a, tick)(c, ids)), host(getattr(b, tick)(c, ids))
            for x, y in zip(oa, ob):
                assert np.array_equal(np.ascontiguousarray(x).view(np.uint8), np.ascontiguousarray(y).view(np.uint8)), (tick, k)
        assert np.array_equal(a.count.cpu().numpy(), b.count.cpu().numpy())
        assert np.array_equal(a.counts.cpu().numpy(), b.counts.cpu().numpy())
        assert int(a.count.item()) + int(a.counts.sum().item()) > 0
        for x in (a, b):
            x.core.close()


def random_settings(rs, n, conf_quantiles=(0.02, 0.3, 0.7)):
    sens = np.r_[0.0, 1.0, 0.5, conf_quantiles][rs.randint(0, 6, n)]
    return sens, np.array(LEVELS, np.int32)[rs.randint(0, 5, n)], np.array(CHUNK_BYTES, np.int32)[rs.randint(0, 6, n)]


@gpu
def test_bank_unrouted_routed_and_ragged():
    """The four-model bank (fused models and the H = 32 model) with settings on slots 0 and 3 only: update_models and
    update_ragged (odd offsets), unrouted and then routed with random masks."""
    m = _mod()
    S = 3000
    rs = np.random.RandomState(13)
    spec = bank_models(m)
    a, b = bank(m, spec, S), bank(m, spec, S)
    rep = Replay(spec)
    for mi in (0, 3):
        ids = rs.permutation(S)[:S - 100].astype(np.int32)
        sens, lvl, chunk = random_settings(rs, len(ids), (0.1, 0.4, 0.6))
        a.set_stream_trigger(mi, sens, lvl, chunk, ids=ids)
        rep.set(mi, ids, sens, lvl, chunk)
    mask = None
    for k in range(16):
        if k == 8:
            mask = rs.randint(0, 256, S).astype(np.uint8)
            mask[:10] = 0
            a.set_stream_models(mask)
        sids = np.arange(S, dtype=np.int32) if k % 4 < 2 else rs.permutation(S)[:S // 2 + 7].astype(np.int32)
        ids = cuda(sids)
        if k % 2 == 0:
            c = cuda(noise((len(sids), CHUNK), rs))
            oa, ob = host(a.update_models(c, ids)), host(b.update_models(c, ids))
        else:
            lens = rs.randint(700, 1400, len(sids))
            offs = cuda((3 + np.concatenate([[0], np.cumsum(lens)])).astype(np.int64))
            pcm = cuda(noise((int(lens.sum()) + 5,), rs))
            oa = host(a.update_ragged(pcm, offs, ids, max_len=1400))
            ob = host(b.update_ragged(pcm, offs, ids, max_len=1400))
        rep.tick(sids, oa, ob[:2], mask)
    print('fired per model', rep.fired)
    assert np.array_equal(a.counts.cpu().numpy(), rep.fired) and rep.fired[[0, 3]].min() > 0
    for x in (a, b):
        x.core.close()


@gpu
def test_one_model_host_and_ragged():
    """One-model handle with settings: update_host with pinned buffers at 64 and 40 streams (zero-copy) and at 200 streams
    (pipelined), update_ragged with odd offsets and update, unrouted and then routed."""
    m = _mod()
    from mycroft_precise_b200.core import pinned_empty, pinned_free
    S = 200
    rs = np.random.RandomState(17)
    spec = [(hot_model(m, seed=5), None, 0.5, 3)]
    a, b = bank(m, spec, S), bank(m, spec, S)
    sens, lvl, chunk = random_settings(rs, S, (0.1, 0.3, 0.5))
    a.set_stream_trigger(0, sens, lvl, chunk)
    rep = Replay(spec)
    rep.set(0, np.arange(S), sens, lvl, chunk)
    pinned = {}

    def pin(name, arr):
        if name not in pinned:
            pinned[name] = pinned_empty(arr.shape, arr.dtype)
        buf = pinned[name][0]
        buf[...] = arr
        return buf

    mask, host_count = None, 0
    for k in range(14):
        if k == 7:
            mask = (rs.randint(0, 2, S) | (rs.randint(0, 128, S) << 1)).astype(np.uint8)
            a.set_stream_models(mask)
        what = ['zc64', 'zc40', 'pipe', 'ragged', 'update'][k % 5]
        if what in ('zc64', 'zc40', 'pipe'):
            n = {'zc64': 64, 'zc40': 40, 'pipe': S}[what]
            sids = np.arange(S, dtype=np.int32)[:n] if what != 'zc40' else np.sort(rs.permutation(S)[:40]).astype(np.int32)
            pcm = noise((n, CHUNK), rs)
            outs = []
            for x, tag in ((a, 'a'), (b, 'b')):
                if what == 'pipe':
                    raw, conf, fired = np.zeros(n, np.float32), np.zeros(n), np.zeros(n, np.uint8)
                    cnt = x.core.update_host(pcm, conf, raw, fired)
                else:
                    raw = pin(tag + what + 'raw', np.zeros(n, np.float32))
                    conf = pin(tag + what + 'conf', np.zeros(n))
                    fired = pin(tag + what + 'fired', np.zeros(n, np.uint8))
                    idp = pin(tag + what + 'ids', sids) if what == 'zc40' else None
                    cnt = x.core.update_host(pin(tag + what + 'pcm', pcm), conf, raw, fired, idp)
                outs.append((raw.copy(), conf.copy(), fired.copy(), cnt))
            rep.tick(sids, outs[0][:3], outs[1][:2], mask)
            assert outs[0][3] == int(outs[0][2].sum())
            host_count += outs[0][3]
            continue
        sids = rs.permutation(S)[:150].astype(np.int32)
        ids = cuda(sids)
        if what == 'ragged':
            lens = rs.randint(600, 1500, len(sids))
            offs = cuda((1 + np.concatenate([[0], np.cumsum(lens)])).astype(np.int64))
            pcm = cuda(noise((int(lens.sum()) + 1,), rs))
            rep.tick(sids, host(a.update_ragged(pcm, offs, ids, max_len=1500)),
                     host(b.update_ragged(pcm, offs, ids, max_len=1500))[:2], mask)
        else:
            c = cuda(noise((len(sids), CHUNK), rs))
            rep.tick(sids, host(a.update(c, ids)), host(b.update(c, ids))[:2], mask)
    print('fired', rep.fired, 'host ticks', host_count)
    assert int(a.count.item()) + int(a.counts[0].item()) + host_count == rep.fired[0] and rep.fired[0] > 0
    for buf, p in pinned.values():
        pinned_free(p)
    for x in (a, b):
        x.core.close()


@gpu
def test_state_rules():
    """A changed setting re-arms mid-stream, an unchanged one keeps the state, clear re-arms and keeps the settings, a mask bit
    0 -> 1 re-arms and keeps them, and a model added after settings exist starts on its own defaults."""
    m = _mod()
    S = 600
    rs = np.random.RandomState(23)
    spec = [(hot_model(m, seed=6), None, 0.5, 3), (hot_model(m, seed=7), None, 0.8, 1)]
    a, b = bank(m, spec, S), bank(m, spec, S)
    rep = Replay(spec)
    cur = {}
    for mi in (0, 1):
        cur[mi] = random_settings(rs, S, (0.05, 0.2, 0.4))
        a.set_stream_trigger(mi, *cur[mi])
        rep.set(mi, np.arange(S), *cur[mi])
    mask = None
    for k in range(18):
        if k == 3:                                                     # new values on some streams, the same on others
            ids = rs.permutation(S)[:200].astype(np.int32)
            sens, lvl, chunk = (x.copy() for x in cur[0])
            sens[ids[:100]] = np.where(sens[ids[:100]] == 1.0, 0.5, 1.0)
            chunk[ids[100:150]] = np.where(chunk[ids[100:150]] == 4096, 3000, 4096)
            a.set_stream_trigger(0, sens[ids], lvl[ids], chunk[ids], ids=ids)
            rep.set(0, ids, sens[ids], lvl[ids], chunk[ids])
            cur[0] = (sens, lvl, chunk)
        if k == 6:
            cl = np.sort(rs.permutation(S)[:150]).astype(np.int32)
            for x in (a, b):
                x.clear(cuda(cl))
            rep.clear(cl)
        if k == 9:
            mask = np.full(S, 0xFF, np.uint8)
            mask[:200] = rs.randint(0, 4, 200)
            a.set_stream_models(mask)
        if k == 12:
            new = mask.copy()
            new[:200] = 0xFF
            a.set_stream_models(new)
            rep.set_masks(mask, new, np.arange(S))
            mask = new
        if k == 14:
            extra = bank_models(m)[1]
            for x in (a, b):
                assert x.add_model(extra[0], extra[1], sensitivity=1.0, trigger_level=0) == 2     # every conf > 0 is hot
            rep.default.append((2 * CHUNK, 1.0, 0))
            rep.fired = np.r_[rep.fired, 0]
            got = a.stream_trigger(2)
            assert np.all(got[0] == 1.0) and np.all(got[1] == 0) and np.all(got[2] == 2048)
        sids = rs.permutation(S)[:S - 50].astype(np.int32)
        c, ids = cuda(noise((len(sids), CHUNK), rs)), cuda(sids)
        rep.tick(sids, host(a.update_models(c, ids)), host(b.update_models(c, ids))[:2], mask)
        if k == 6:                                                     # clear kept the settings
            got = a.stream_trigger(0)
            assert np.array_equal(got[0].view(np.uint64), cur[0][0].view(np.uint64)) and np.array_equal(got[2], cur[0][2])
    print('fired per model', rep.fired)
    assert np.array_equal(a.counts.cpu().numpy(), rep.fired) and rep.fired.min() > 0
    for x in (a, b):
        x.core.close()


@gpu
def test_stream_trigger_api():
    m = _mod()
    c = m.PreciseB200(max_streams=16, sensitivity=0.25, trigger_level=2, chunk_samples=512)
    sens, lvl, chunk = c.stream_trigger(0)
    assert sens.dtype == np.float64 and lvl.dtype == np.int32 and chunk.dtype == np.int32
    assert np.all(sens == 0.25) and np.all(lvl == 2) and np.all(chunk == 1024)
    odd = np.array([0x7ff8000000000123, 0x8000000000000000, 0x7e37e43c8800759c], np.uint64).view(np.float64)  # NaN, -0.0, 1e300
    ids = np.array([2, 9, 15], np.int32)
    c.set_stream_trigger(0, odd, np.array([-2 ** 31, 2 ** 31 - 1, 0]), np.array([1, 2 ** 31 - 1, 3000]), ids=ids)

    def snapshot():
        return tuple(x.copy() for x in c.stream_trigger(0))

    want = snapshot()
    assert np.array_equal(want[0][ids].view(np.uint64), odd.view(np.uint64))
    assert list(want[1][ids]) == [-2 ** 31, 2 ** 31 - 1, 0] and list(want[2][ids]) == [1, 2 ** 31 - 1, 3000]
    rest = np.setdiff1d(np.arange(16), ids)
    assert np.all(want[0][rest] == 0.25) and np.all(want[1][rest] == 2) and np.all(want[2][rest] == 1024)
    got = c.stream_trigger(0, np.array([15, 2], np.int32))
    assert np.array_equal(got[2], [3000, 1])
    bad = [dict(slot=1), dict(slot=-1), dict(chunk=0), dict(chunk=-5), dict(ids=[3, 3]), dict(ids=[3, 16]), dict(ids=[-1, 3]),
           dict(ids=None, n=17)]
    for case in bad:
        n = case.get('n', 2)
        i = case.get('ids', [4, 5])
        i = None if i is None else np.array(i, np.int32)
        s, l, ch = np.full(n, 0.7), np.full(n, 1, np.int32), np.full(n, case.get('chunk', 2048), np.int32)
        with pytest.raises(ValueError):
            c.set_stream_trigger(case.get('slot', 0), s, l, ch, ids=i)
        vp = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)   # noqa: E731
        assert c.lib.pb_set_stream_trigger(c._h, case.get('slot', 0), vp(i), vp(s), vp(l), vp(ch), n) == -1, case
        now = snapshot()
        assert all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(now, want)), case
    s1 = np.zeros(1)
    assert c.lib.pb_set_stream_trigger(c._h, 0, None, s1.ctypes.data_as(C.c_void_p), None, None, 1) == -1
    assert c.lib.pb_set_stream_trigger(c._h, 0, None, None, None, None, -1) == -1
    assert c.lib.pb_get_stream_trigger(c._h, 1, None, 1, None, None, None) == -1
    with pytest.raises(ValueError):
        c.stream_trigger(1)
    with pytest.raises(ValueError):
        c.stream_trigger(0, np.array([16], np.int32))
    with pytest.raises(ValueError):
        c.set_stream_trigger(0, 0.5, 1.5, 2048)                       # a float trigger level
    with pytest.raises(ValueError):
        c.set_stream_trigger(0, 0.5, 2 ** 31, 2048)                   # outside int32
    with pytest.raises(ValueError):
        c.set_stream_trigger(0, np.full(3, 0.5), 1, np.full(4, 2048))  # lengths differ
    assert all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(snapshot(), want))
    c.set_stream_trigger(0, 0.5, 3, 4096, ids=np.array([4], np.int32))
    assert [x[4] for x in c.stream_trigger(0)] == [0.5, 3, 4096]
    c.close()


def test_stream_trigger_null_handle_is_invalid():
    import os
    import __graft_entry__ as g
    from mycroft_precise_b200.core import lib_path, get_lib
    if not os.path.isfile(lib_path()):
        g.build()
    lib = get_lib()
    ids = np.arange(4, dtype=np.int32)
    sens, lvl, chunk = np.full(4, 0.5), np.zeros(4, np.int32), np.full(4, 2048, np.int32)
    p = [a.ctypes.data_as(C.c_void_p) for a in (ids, sens, lvl, chunk)]
    assert lib.pb_set_stream_trigger(None, 0, p[0], p[1], p[2], p[3], 4) == -1 and b'null' in lib.pb_last_error()
    assert lib.pb_get_stream_trigger(None, 0, p[0], 4, p[1], p[2], p[3]) == -1
    assert lib.pb_set_stream_trigger(None, 0, None, None, None, None, 0) == -1
    assert lib.pb_get_stream_trigger(None, 0, None, 0, None, None, None) == -1
