"""Stream audio history (pb_set_history, pb_set_stream_history, pb_read_history): every tick entry point, the on / off and
restart rules, no effect on outputs, activation clips and the API.

-m gpu, except the C-ABI null-handle check at the end.  The oracle is exact: each stream's fed int16 audio concatenated in
numpy, zeros before the stream's history start.  Every read must equal it bit for bit.
"""
import ctypes as C

import numpy as np
import pytest

from test_gpu_model_bank import bank_models
from test_gpu_stream_models import bank, cuda, host, noise
from test_gpu_stream_trigger import hot_model

gpu = pytest.mark.gpu
CHUNK = 1024


def _mod():
    import mycroft_precise_b200 as m
    return m


class Audio:
    """What each stream was fed (its last `keep` samples while it has history), its sample count and history start."""

    def __init__(self, S, keep):
        self.keep = keep
        self.buf = {}
        self.n = np.zeros(S, np.int64)
        self.start = np.zeros(S, np.int64)
        self.on = np.zeros(S, bool)

    def feed(self, sid, x):
        if self.on[sid]:
            self.buf[sid] = np.concatenate([self.buf.get(sid, np.zeros(0, np.int16)), x])[-self.keep:]
        self.n[sid] += len(x)

    def feed_rows(self, sids, pcm):
        for sid, x in zip(sids, pcm):
            self.feed(int(sid), x)

    def switch(self, sids, on):
        for sid, o in zip(sids, np.broadcast_to(on, len(sids))):
            if o and not self.on[sid]:
                self.start[sid] = self.n[sid]
                self.buf[sid] = np.zeros(0, np.int16)
            self.on[sid] = bool(o)

    def restart(self, sids, n):
        """pb_clear (n = 0) or pb_import_streams (n = the record's n_samples)."""
        for sid, v in zip(sids, np.broadcast_to(n, len(sids))):
            self.n[sid] = self.start[sid] = v
            self.buf[sid] = np.zeros(0, np.int16)

    def expect(self, sids, samples):
        out = np.zeros((len(sids), samples), np.int16)
        for r, sid in enumerate(sids):
            if not self.on[sid]:
                continue
            m = min(samples, int(self.n[sid] - self.start[sid]))
            if m > 0:
                out[r, samples - m:] = self.buf[sid][-m:]
        return out


def check_reads(sb, audio, sids, sizes):
    for samples in sizes:
        got = sb.read_history(cuda(np.asarray(sids, np.int32)), samples).cpu().numpy()
        want = audio.expect(sids, samples)
        bad = np.nonzero((got != want).any(1))[0]
        assert bad.size == 0, 'samples %d: %d rows differ, first stream %d' % (samples, bad.size, sids[bad[0]])


@gpu
@pytest.mark.parametrize('S', [7, 9000])
@pytest.mark.parametrize('H', [24000, 5001])
def test_update(S, H):
    """Permuted and partial ticks, a random subset of streams on, enough ticks to wrap the rows three times; reads of every
    length class (full, shorter, one sample), of streams on and off."""
    m = _mod()
    rs = np.random.RandomState(S + H)
    sb = m.StreamBatch(m.GruModel.random(13, 20, seed=0, scale=0.1), S)
    sb.set_history(H)
    on = rs.rand(S) < 0.5
    on[0] = True
    sb.set_stream_history(on)
    assert np.array_equal(sb.stream_history(), on)
    audio = Audio(S, H)
    audio.switch(np.arange(S), on)
    K = 5 * H // CHUNK + 3                                             # a stream misses at most a third of the ticks
    probe = np.arange(S) if S < 100 else rs.permutation(S)[:700]
    for k in range(K):
        sids = rs.permutation(S)[:S if k % 3 else S // 2 + 1].astype(np.int32)
        pcm = noise((len(sids), CHUNK), rs)
        sb.update(cuda(pcm), cuda(sids))
        audio.feed_rows(sids, pcm)
        if k % 16 == 15 or k == K - 1:
            check_reads(sb, audio, probe, [H, 777, 1] if k == K - 1 else [H])
    assert audio.n.min() > 3 * H                                       # every row wrapped at least three times
    sb.core.close()


@gpu
def test_update_models_routed():
    """A four-model bank, routed, some streams with mask 0: they still consume audio, so they still append."""
    m = _mod()
    S, H = 300, 5001
    rs = np.random.RandomState(2)
    sb = bank(m, bank_models(m), S)
    masks = rs.randint(0, 16, S).astype(np.uint8)
    masks[:40] = 0
    sb.set_stream_models(masks)
    sb.set_history(H, max_rows=250)
    on = np.zeros(S, bool)
    on[rs.permutation(S)[:230]] = True
    on[:20] = True
    sb.set_stream_history(on)
    audio = Audio(S, H)
    audio.switch(np.arange(S), on)
    for k in range(14):
        sids = rs.permutation(S)[:S if k % 2 else 201].astype(np.int32)
        pcm = noise((len(sids), CHUNK), rs)
        sb.update_models(cuda(pcm), cuda(sids))
        audio.feed_rows(sids, pcm)
    check_reads(sb, audio, np.arange(S), [H, 4000])
    sb.core.close()


@gpu
@pytest.mark.parametrize('generic', [False, True])
def test_update_ragged(generic):
    """Odd offsets, lengths from 1 to 30 000 (above history_samples: only the last 24 000 survive), then uniform ticks on the
    now-ragged handle."""
    m = _mod()
    S, H = 64, 24000
    rs = np.random.RandomState(5 + generic)
    sb = m.StreamBatch(m.GruModel.random(13, 20, seed=1, scale=0.1), S)
    if generic:
        sb.core.force_generic(True)
    sb.set_history(H)
    on = rs.rand(S) < 0.7
    sb.set_stream_history(on)
    audio = Audio(S, H)
    audio.switch(np.arange(S), on)
    for k in range(8):
        n = S if k % 2 else 40
        sids = rs.permutation(S)[:n].astype(np.int32)
        if k % 4 == 0:
            lens = rs.randint(1, 30001, n)
            lens[:3] = [1, 30000, H + 1][:min(3, n)]
        else:
            lens = rs.randint(1, 3000, n)
        off = np.concatenate([[3], 3 + np.cumsum(lens)]).astype(np.int64)
        flat = noise((int(off[-1]) + 5,), rs)
        sb.update_ragged(cuda(flat), cuda(off), cuda(sids))
        for j, sid in enumerate(sids):
            audio.feed(int(sid), flat[off[j]:off[j + 1]])
        check_reads(sb, audio, np.arange(S), [H])
    for k in range(30):
        sids = rs.permutation(S)[:S if k % 2 else 33].astype(np.int32)
        pcm = noise((len(sids), CHUNK), rs)
        sb.update(cuda(pcm), cuda(sids))
        audio.feed_rows(sids, pcm)
    check_reads(sb, audio, np.arange(S), [H, 1001, 1])
    sb.core.close()


@gpu
@pytest.mark.parametrize('S', [40, 200, 40000])
def test_update_vectors_and_host(S):
    """update_vectors, then update_host: zero-copy at 40 streams (pinned buffers), pipelined at 200 and at 40 000 (three
    sub-batches)."""
    m = _mod()
    from mycroft_precise_b200.core import pinned_empty, pinned_free
    H = 5001
    rs = np.random.RandomState(S)
    sb = m.StreamBatch(m.GruModel.random(13, 20, seed=2, scale=0.1), S)
    sb.set_history(H)
    on = np.arange(S) % 3 == 0
    sb.set_stream_history(on)
    audio = Audio(S, H)
    audio.switch(np.arange(S), on)
    for k in range(3):
        sids = rs.permutation(S).astype(np.int32)
        pcm = noise((S, CHUNK), rs)
        sb.core.update_vectors(cuda(pcm), cuda(sids))
        audio.feed_rows(sids, pcm)
    pcm_h, p1 = pinned_empty((S, CHUNK), np.int16)
    conf_h, p2 = pinned_empty((S,), np.float64)
    try:
        for k in range(6):
            pcm_h[:] = noise((S, CHUNK), rs)
            sb.update_host(pcm_h, conf_h)
            audio.feed_rows(np.arange(S), pcm_h.copy())
    finally:
        pinned_free(p1)
        pinned_free(p2)
    probe = np.arange(S) if S <= 200 else np.concatenate([np.arange(0, S, 3)[:1500], rs.permutation(S)[:500]])
    check_reads(sb, audio, probe, [H, 2048])
    sb.core.close()


@gpu
def test_switching_and_restarts():
    """On mid-stream, off and on again, clear, import into streams that are on (at other ids), max_rows exceeded, reads of
    streams that are off, set_history again and freed."""
    m = _mod()
    S, H, R = 50, 3001, 20
    rs = np.random.RandomState(9)
    sb = m.StreamBatch(m.GruModel.random(13, 20, seed=3, scale=0.1), S)
    with pytest.raises(m.PBError):
        sb.read_history()
    with pytest.raises(m.PBError):
        sb.set_stream_history(True)
    assert not sb.stream_history().any()
    sb.set_history(H, max_rows=R)
    audio = Audio(S, H)

    def tick(K=2, sids=None):
        for _ in range(K):
            s = np.arange(S, dtype=np.int32) if sids is None else sids
            pcm = noise((len(s), CHUNK), rs)
            sb.update(cuda(pcm), cuda(s))
            audio.feed_rows(s, pcm)

    def switch(ids, on):
        ids = np.asarray(ids, np.int32)
        sb.set_stream_history(on, ids)
        audio.switch(ids, on)

    def verify():
        assert np.array_equal(sb.stream_history(), audio.on)
        check_reads(sb, audio, np.arange(S), [audio.keep, 1500])

    switch(np.arange(10), True)
    tick(3)
    verify()
    switch(np.arange(10, 15), np.ones(5, bool))                  # mid-stream: they start empty
    tick(2)
    verify()
    switch([3], False)
    verify()
    switch([3, 4], [True, True])                                 # 3 starts empty again, 4 keeps its audio
    tick(1)
    verify()
    sb.clear(cuda(np.array([5, 6, 30], np.int32)))
    audio.restart([5, 6, 30], 0)
    tick(1, np.array([5, 30, 1], np.int32))
    verify()
    src, dst = np.array([20, 21], np.int32), np.array([7, 8], np.int32)
    state = sb.core.export_streams(cuda(src))
    sb.core.import_streams(state, dst)
    audio.restart(dst, audio.n[src])
    verify()
    tick(2)
    verify()
    before = sb.read_history().cpu().numpy()
    with pytest.raises(ValueError):
        sb.set_stream_history(True, np.arange(15, 40, dtype=np.int32))       # 15 on + 25 > 20 rows
    with pytest.raises(ValueError):
        sb.set_stream_history([True, False], np.array([40, 40], np.int32))
    with pytest.raises(ValueError):
        sb.set_stream_history(True, np.array([S], np.int32))
    assert np.array_equal(sb.stream_history(), audio.on)
    assert np.array_equal(sb.read_history().cpu().numpy(), before)
    assert not before[~audio.on].any()
    switch(np.arange(15, 20), True)                              # exactly max_rows
    tick(1)
    verify()
    with pytest.raises(ValueError):
        sb.read_history(samples=H + 1)
    with pytest.raises(ValueError):
        sb.read_history(samples=0)
    sb.set_history(2000, max_rows=5)                             # a new pool: every stream off
    n = audio.n
    audio = Audio(S, 2000)
    audio.n = n
    verify()
    assert not sb.read_history().cpu().numpy().any()
    switch([1, 2], True)
    tick(3)
    verify()
    sb.set_history(0, 0)
    assert not sb.stream_history().any()
    with pytest.raises(m.PBError):
        sb.read_history(samples=10)
    tick(1)
    sb.core.close()


def records(sb, S):
    return sb.core.export_streams(cuda(np.arange(S, dtype=np.int32))).cpu().numpy()


@gpu
def test_no_effect_on_outputs():
    """The same ticks (update, update_models, update_ragged, clear, import) on a bank with history on every stream and on one
    without: raw, conf, fired, counts and state records bit-identical."""
    m = _mod()
    S = 500
    rs = np.random.RandomState(11)
    spec = [(hot_model(m), None, 0.5, 3), (hot_model(m, seed=9), None, 0.5, 1)]
    a, b = bank(m, spec, S), bank(m, spec, S)
    a.set_history()
    a.set_stream_history(True)
    for k in range(16):
        sids = rs.permutation(S)[:S if k % 2 else 301].astype(np.int32)
        if k % 5 == 4:
            lens = rs.randint(1, 3000, len(sids))
            off = np.concatenate([[1], 1 + np.cumsum(lens)]).astype(np.int64)
            flat = noise((int(off[-1]) + 1,), rs)
            oa = host(a.update_ragged(cuda(flat), cuda(off), cuda(sids)))
            ob = host(b.update_ragged(cuda(flat), cuda(off), cuda(sids)))
        else:
            pcm = noise((len(sids), CHUNK), rs)
            oa = host(a.update_models(cuda(pcm), cuda(sids)))
            ob = host(b.update_models(cuda(pcm), cuda(sids)))
        for x, y in zip(oa, ob):
            assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), k
        if k == 8:
            for x in (a, b):
                x.clear(cuda(np.arange(10, dtype=np.int32)))
                x.core.import_streams(x.core.export_streams(cuda(np.arange(20, 30, dtype=np.int32))),
                                      np.arange(30, 40, dtype=np.int32))
    assert np.array_equal(a.counts.cpu().numpy(), b.counts.cpu().numpy()) and int(a.counts.sum()) > 0
    assert np.array_equal(records(a, S), records(b, S))
    for x in (a, b):
        x.core.close()


@gpu
def test_activation_audio():
    """A bank of hot models, history on most streams: every fired (model, item) pair of a stream with history appears in
    nonzero order, and its clip is the last buffer_samples samples ending with the firing tick's chunk."""
    m = _mod()
    S = 200
    rs = np.random.RandomState(13)
    sb = bank(m, [(hot_model(m), None, 0.5, 1), (hot_model(m, seed=5), None, 0.5, 2)], S)
    B = sb.pr.buffer_samples
    sb.set_history()
    on = rs.rand(S) < 0.75
    sb.set_stream_history(on)
    audio = Audio(S, B)
    audio.switch(np.arange(S), on)
    pairs_seen = 0
    for k in range(30):
        sids = rs.permutation(S)[:S if k % 2 else 120].astype(np.int32)
        pcm = noise((len(sids), CHUNK), rs)
        out = sb.update_models(cuda(pcm), cuda(sids))
        audio.feed_rows(sids, pcm)
        got = sb.activation_audio(out['fired'], cuda(sids))
        fired = out['fired'].cpu().numpy()
        want = [(mi, sids[i]) for mi, i in zip(*np.nonzero(fired)) if on[sids[i]]]
        assert [(int(a), int(b)) for a, b in zip(got['slot'].cpu().numpy(), got['stream'].cpu().numpy())] == \
            [(int(a), int(b)) for a, b in want], k
        clip = got['audio'].cpu().numpy()
        assert clip.shape == (len(want), B)
        if want:
            assert np.array_equal(clip, audio.expect([s for _, s in want], B)), k
        one = sb.activation_audio(out['fired'][0], cuda(sids), samples=CHUNK)     # [n] form, the last chunk only
        w0 = [s for mi, s in want if mi == 0]
        assert one['audio'].shape == (len(w0), CHUNK)
        if w0:
            idx = [int(np.nonzero(sids == s)[0][0]) for s in w0]
            assert np.array_equal(one['audio'].cpu().numpy(), pcm[idx])
        pairs_seen += len(want)
    assert pairs_seen > 20
    sb.core.close()


def test_history_null_handle_is_invalid():
    import os
    import __graft_entry__ as g
    from mycroft_precise_b200.core import lib_path, get_lib
    if not os.path.isfile(lib_path()):
        g.build()
    lib = get_lib()
    buf = np.zeros(64, np.uint8)
    p = buf.ctypes.data_as(C.c_void_p)
    assert lib.pb_set_history(None, 100, 1) == -1 and b'null' in lib.pb_last_error()
    assert lib.pb_set_history(None, 0, 0) == -1
    assert lib.pb_set_stream_history(None, None, p, 4) == -1
    assert lib.pb_set_stream_history(None, None, None, 0) == -1
    assert lib.pb_get_stream_history(None, None, 4, p) == -1
    assert lib.pb_read_history(None, None, 1, 10, p, None) == -1
    assert lib.pb_read_history(None, None, 0, 10, None, None) == -1
