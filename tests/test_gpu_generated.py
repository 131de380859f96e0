"""Generated training audio on the device (pb_generate; PreciseB200.generate, offline.Generator / train_generated,
python -m mycroft_precise_b200.train_generated) against oracle/generated.py's exact restatement, pb_mfcc, the oracle
listener and the float64 training oracle.  -m gpu."""
import os
import sys
import wave

import numpy as np
import pytest

from oracle import generated as og
from oracle import train as ot
from oracle.listener import OracleListener
from oracle.params import OracleParams

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import train_task  # noqa: E402

gpu = pytest.mark.gpu


def _sig(n, seed, sigma=3000):
    rs = np.random.RandomState(seed)
    return np.clip(np.round(rs.randn(n) * sigma), -32768, 32767).astype(np.int16)


def _offs(recs):
    return np.concatenate([[0], np.cumsum([len(r) for r in recs])]).astype(np.int64)


class Fixture:
    def __init__(self):
        import torch
        import mycroft_precise_b200 as m
        from mycroft_precise_b200.core import GEN_ITEM, GEN_SEGMENT
        self.m, self.torch, self.GEN_ITEM, self.GEN_SEGMENT = m, torch, GEN_ITEM, GEN_SEGMENT
        self.core = m.PreciseB200()

    def dev(self, recs, lead=0):
        """Recordings back to back after `lead` samples: (tensor, offsets of the recordings)."""
        a = np.concatenate([_sig(lead, 999)] + list(recs) + [np.zeros(0, np.int16)])
        return self.torch.from_numpy(a).cuda(), _offs(recs) + lead

    def tables(self, items, segs):
        it = np.zeros(len(items), self.GEN_ITEM)
        for i, (b, f, L, s0, s1) in enumerate(items):
            it[i] = (b, 0, f, L, s0, s1)
        sg = np.zeros(len(segs), self.GEN_SEGMENT)
        for j, (c, a, n) in enumerate(segs):
            sg[j] = (c, 0, a, n)
        return it, sg


@pytest.fixture(scope='module')
def fx():
    pytest.importorskip('torch')
    f = Fixture()
    yield f
    f.core.close()


def _case():
    bgs = [_sig(100003, 1, 2000), _sig(5000, 2, 300), np.zeros(4000, np.int16), np.full(64, 30000, np.int16), _sig(3, 3)]
    clips = [_sig(n, 10 + i, 1500 + 500 * i) for i, n in enumerate([1, 7, 511, 1600, 4097, 30001, 100001])]
    clips.append(np.zeros(900, np.int16))                                      # a silent clip
    clips.append(np.asarray([32767] + [1] * 63, np.int16))                     # all its energy in one sample: saturates
    items, segs = [], []

    def item(b, f, L, parts):
        s0 = len(segs)
        segs.extend(parts)
        items.append((b, f, L, s0, len(segs)))
    for L in (1, 2, 7, 8, 511, 4096, 33333, 100000):                          # lengths at odd clip offsets
        item(0, 0.4 if L % 2 else 0.9, L, [(6, 1, min(L, 60000)), (-1, 0, 17), (5, 1, 30000), (4, 5, 4092), (6, 11, 50000)])
    item(1, 0.9, 5000, [(-1, 0, 6000)])                                        # silence only
    item(2, 0.7, 4000, [(3, 0, 1600), (7, 0, 900), (-1, 0, 3000)])            # silent background and a silent clip
    item(3, 0.9, 64, [(8, 0, 64)])                                             # saturation
    item(1, 0.4, 0, [])                                                        # empty
    for r in range(40):                                                        # many items, repeated clips
        item(r % 2, 0.4 + 0.5 * r / 40, 999 + 37 * r, [(2, 0, 511), (2, 100, 400), (-1, 0, 64), (4, 7, 4000)])
    return bgs, clips, items, segs


@gpu
def test_streams_are_the_exact_oracle(fx):
    bgs, clips, items, segs = _case()
    bg, bo = fx.dev(bgs, 5)
    cl, co = fx.dev(clips, 3)
    it, sg = fx.tables(items, segs)
    out, x = fx.core.generate(bg, bo, cl, co, it, sg)
    assert x is None
    got = out.cpu().numpy()
    want = og.exact(bgs, clips, items, segs)
    o = _offs(want)
    for i, w in enumerate(want):
        assert got[o[i]:o[i + 1]].tobytes() == w.tobytes(), i
    assert got.shape[0] == o[-1]
    assert (want[10] == 32767).any()                                          # the saturating item


def _frames_window(core, stream, n, T):
    """The listener window after n samples of the stream: pb_mfcc's last T frames of its first n samples."""
    torch = core.torch
    f = core.mfcc(torch.from_numpy(stream[:n].copy()).cuda()[None])[0].cpu().numpy()
    w = np.zeros((T, f.shape[1]), np.float32)
    if f.shape[0]:
        w[T - min(T, f.shape[0]):] = f[-T:]
    return w


@gpu
@pytest.mark.parametrize('generic', [False, True])
def test_inputs_are_pb_mfcc_of_the_streams(fx, generic):
    bgs = [_sig(60000, 4, 1200), _sig(9000, 5, 700)]
    clips = [_sig(12000, 6, 2500), _sig(3001, 7, 1800)]
    items = [(0, 0.6, 40960, 0, 3), (1, 0.45, 8192, 3, 5), (0, 0.8, 2048, 5, 6)]
    segs = [(0, 0, 12000), (-1, 0, 26000), (1, 1, 3000), (1, 0, 3001), (-1, 0, 6000), (0, 3, 2048)]
    bg, bo = fx.dev(bgs, 8)
    cl, co = fx.dev(clips, 1)
    it, sg = fx.tables(items, segs)
    wins = np.asarray([(0, 0), (0, 1), (0, 19), (1, 3), (0, 7), (2, 0), (1, 0), (0, 19)], np.int64)
    fx.core.force_generic(generic)
    try:
        out, x = fx.core.generate(bg, bo, cl, co, it, sg, wins, chunk=2048, divisor=32768)
        streams = og.exact(bgs, clips, items, segs)
        assert out.cpu().numpy().tobytes() == np.concatenate(streams).tobytes()
        got = x.cpu().numpy()
        T = fx.core.n_features
        for w, (i, c) in enumerate(wins):
            want = _frames_window(fx.core, streams[i], (c + 1) * 2048, T)
            assert got[w].tobytes() == want.tobytes(), (w, i, c)
        assert not got[5][:T - 1].any() and got[5][T - 1].any()               # one frame: zero rows before it
    finally:
        fx.core.force_generic(False)


@gpu
def test_inputs_at_load_audio_scale_follow_the_oracle_listener(fx):
    bgs = [_sig(50000, 8, 1000)]
    clips = [_sig(16000, 9, 3000)]
    items = [(0, 0.7, 49152, 0, 3)]
    segs = [(-1, 0, 8000), (0, 0, 16000), (-1, 0, 40000)]
    bg, bo = fx.dev(bgs)
    cl, co = fx.dev(clips)
    it, sg = fx.tables(items, segs)
    n = 49152 // 2048
    wins = np.asarray([(0, c) for c in range(n)], np.int64)
    out, x = fx.core.generate(bg, bo, cl, co, it, sg, wins, chunk=2048, divisor=32767)
    stream = out.cpu().numpy()
    lis = OracleListener(None, OracleParams(), 2048)
    got = x.cpu().numpy()
    for c in range(n):
        want = lis.update_vectors(stream[c * 2048:(c + 1) * 2048].astype(np.float32) / np.float32(32767))
        assert np.allclose(got[c], want, rtol=1e-4, atol=1e-3), (c, np.max(np.abs(got[c] - want)))   # vectorize's bound


@gpu
def test_split_calls_equal_one_call(fx):
    bgs, clips, items, segs = _case()
    bg, bo = fx.dev(bgs)
    cl, co = fx.dev(clips)
    it, sg = fx.tables(items, segs)
    wins = np.asarray([(i, c) for i, t in enumerate(items) for c in range(0, t[2] // 1024, 3)], np.int64)
    out, x = fx.core.generate(bg, bo, cl, co, it, sg, wins, chunk=1024)
    outs, xs = [], []
    for a, b in ((0, 7), (7, 12), (12, len(items))):
        sub = [(bb, f, L, s0, s1) for bb, f, L, s0, s1 in items[a:b]]
        ti, ts = fx.tables(sub, segs)
        w = wins[(wins[:, 0] >= a) & (wins[:, 0] < b)] - np.asarray([a, 0])
        o, y = fx.core.generate(bg, bo, cl, co, ti, ts, w, chunk=1024)
        outs.append(o.cpu().numpy())
        xs.append(y.cpu().numpy())
    assert np.concatenate(outs).tobytes() == out.cpu().numpy().tobytes()
    assert np.concatenate(xs).tobytes() == x.cpu().numpy().tobytes()


@gpu
def test_refusals_change_nothing(fx):
    torch = fx.torch
    bgs, clips, items, segs = _case()
    bg, bo = fx.dev(bgs)
    cl, co = fx.dev(clips)
    it, sg = fx.tables(items[:3], segs)
    lib, core = fx.core.lib, fx.core
    from mycroft_precise_b200.core import _ptr, _np_ptr
    out = torch.full((300000,), 7, dtype=torch.int16, device='cuda')
    x = torch.full((4, core.n_features, core.feature_size), 7.0, device='cuda')

    def call(items=it, segs=sg, wins=np.asarray([(0, 0)], np.int64), chunk=1, divisor=32767, d_out=out, d_in=x, bgo=bo):
        return lib.pb_generate(core._h, _ptr(bg), _np_ptr(bgo), len(bgo) - 1, _ptr(cl), _np_ptr(co), len(co) - 1,
                               _np_ptr(items), len(items), _np_ptr(segs), len(segs), _np_ptr(wins), len(wins), chunk,
                               divisor, _ptr(d_out), _ptr(d_in), None)
    bad = []
    b = it.copy(); b[0]['background'] = len(bgs); bad.append(dict(items=b))
    b = it.copy(); b[0]['gain'] = float('nan'); bad.append(dict(items=b))
    b = it.copy(); b[0]['gain'] = -0.1; bad.append(dict(items=b))
    b = it.copy(); b[0]['length'] = len(bgs[0]) + 1; bad.append(dict(items=b))
    b = it.copy(); b[2]['seg_begin'] = b[2]['seg_end']; bad.append(dict(items=b))             # segments too short
    b = it.copy(); b[0]['seg_end'] = len(sg) + 1; bad.append(dict(items=b))
    s = sg.copy(); s[0]['clip'] = len(clips); bad.append(dict(segs=s))
    s = sg.copy(); s[0]['start'] = len(clips[s[0]['clip']]); bad.append(dict(segs=s))
    s = sg.copy(); s[1]['start'] = 1; bad.append(dict(segs=s))                                  # silence with a start
    s = sg.copy(); s[1]['length'] = 2 ** 62 + 1; bad.append(dict(segs=s))                       # longer than 2^62
    bad += [dict(wins=np.asarray([(3, 0)], np.int64)), dict(wins=np.asarray([(0, 1)], np.int64)),
            dict(wins=np.asarray([(0, 0)], np.int64), d_in=None), dict(d_out=None, d_in=None), dict(divisor=1000),
            dict(chunk=0), dict(bgo=bo[::-1].copy())]
    for kw in bad:
        rc = call(**kw)
        assert rc == -1, (kw, rc)
    torch.cuda.synchronize()
    assert (out == 7).all() and (x == 7).all()
    assert call() == 0


@gpu
def test_items_sharing_segment_ranges(fx):
    """Items may share or overlap segment ranges at different lengths: each reads the range from its own sample 0."""
    bgs = [_sig(20000, 31, 900), _sig(7000, 32, 2000)]
    clips = [_sig(4000, 33, 2500), _sig(3001, 34, 1500)]
    segs = [(-1, 0, 1000), (0, 0, 4000), (1, 1, 3000), (-1, 0, 2 ** 62), (0, 7, 3993)]
    items = [(0, 0.9, 5000, 0, 2), (0, 0.4, 100, 0, 2), (1, 0.6, 7000, 1, 4), (0, 0.7, 12000, 0, 4), (1, 0.5, 3000, 2, 5),
             (0, 0.8, 4000, 1, 2), (1, 0.45, 6999, 0, 5)]
    bg, bo = fx.dev(bgs, 1)
    cl, co = fx.dev(clips, 2)
    it, sg = fx.tables(items, segs)
    wins = np.asarray([(i, c) for i, t in enumerate(items) for c in range(t[2] // 1000)], np.int64)
    out, x = fx.core.generate(bg, bo, cl, co, it, sg, wins, chunk=1000)
    want = og.exact(bgs, clips, items, segs)
    assert out.cpu().numpy().tobytes() == np.concatenate(want).tobytes()
    assert (want[0][1000:5000] != want[1][0]).any()                            # the clip is there, not silence
    alone = []                                                                  # the same items, one call each
    for i, t in enumerate(items):
        ti, ts = fx.tables([t], segs)
        o, y = fx.core.generate(bg, bo, cl, co, ti, ts, wins[wins[:, 0] == i] * np.asarray([0, 1]), chunk=1000)
        alone.append(y.cpu().numpy())
    assert np.concatenate(alone).tobytes() == x.cpu().numpy().tobytes()


@gpu
def test_unsupported_front_end_and_untouched_state(fx):
    m, torch, lib = fx.m, fx.torch, fx.core.lib
    from mycroft_precise_b200.core import _ptr, _np_ptr
    bgs, clips, items, segs = _case()
    it, sg = fx.tables(items[:3], segs)
    wins = np.asarray([(2, 0)], np.int64)
    # d_inputs on a front end outside the fused family
    core2 = m.PreciseB200(m.ListenerParams(use_delta=True))
    bg, bo = fx.dev(bgs)
    cl, co = fx.dev(clips)
    x = torch.full((1, core2.n_features, core2.feature_size), 7.0, device='cuda')
    assert lib.pb_generate(core2._h, _ptr(bg), _np_ptr(bo), len(bo) - 1, _ptr(cl), _np_ptr(co), len(co) - 1, _np_ptr(it),
                           len(it), _np_ptr(sg), len(sg), _np_ptr(wins), 1, 1, 32767, None, _ptr(x), None) == -2
    o, _ = core2.generate(bg, bo, cl, co, it, sg)                              # d_out alone is fine there
    torch.cuda.synchronize()
    assert (x == 7).all() and o.cpu().numpy().tobytes() == np.concatenate(og.exact(bgs, clips, items[:3], segs)).tobytes()
    core2.close()
    # stream state and the pool, after refused and accepted calls
    g = m.GruModel.random(13, 20, seed=8, scale=0.1)
    sb = m.StreamBatch(g, 3)
    sb.set_pool(1)
    sb.pool_load(0, g)
    sb.set_stream_pool(np.zeros(3, np.int32))
    rs = np.random.RandomState(1)
    pcm = torch.from_numpy(np.clip(rs.randn(3, 1024) * 3000, -32768, 32767).astype(np.int16)).cuda()
    sb.update_pool(pcm)
    core = sb.core
    before = core.export_streams(n=3).cpu().numpy()
    ids = core.stream_pool()
    bad = it.copy()
    bad[0]['gain'] = -1.0
    with pytest.raises(Exception):
        core.generate(bg, bo, cl, co, bad, sg, wins, chunk=1)
    core.generate(bg, bo, cl, co, it, sg, wins, chunk=1)
    torch.cuda.synchronize()
    assert core.export_streams(n=3).cpu().numpy().tobytes() == before.tobytes()
    assert np.array_equal(core.stream_pool(), ids)
    a = sb.update_pool(pcm)['raw'].cpu().numpy()
    ref = m.StreamBatch(g, 3)
    ref.set_pool(1)
    ref.pool_load(0, g)
    ref.set_stream_pool(np.zeros(3, np.int32))
    ref.update_pool(pcm)
    assert ref.update_pool(pcm)['raw'].cpu().numpy().tobytes() == a.tobytes()


@gpu
def test_generator_plans_what_the_device_makes(fx):
    from mycroft_precise_b200.offline import Generator
    rs = np.random.RandomState(1)
    bgs = [_sig(int(n), 20 + i, 800) for i, n in enumerate(rs.randint(20000, 90000, 5))]
    wake = [_sig(int(n), 40 + i, 3000) for i, n in enumerate(rs.randint(8000, 16000, 3))]
    other = [_sig(int(n), 60 + i, 2000) for i, n in enumerate(rs.randint(4000, 16000, 3))]
    gen = Generator(fx.core, bgs, wake, other, chunk=2048, seed=3)
    plan = gen.plan(300)
    x, tg, audio, ends = gen.run(plan, out=True)
    assert x.shape[0] == 300 == tg.shape[0] == ends.shape[0]
    items, segs, wins, tg2 = gen.tables(plan)
    streams = og.exact(bgs, wake + other, [(r['background'], r['gain'], r['length'], r['seg_begin'], r['seg_end'])
                                            for r in items], [(s['clip'], s['start'], s['length']) for s in segs])
    assert audio.cpu().numpy().tobytes() == np.concatenate(streams).tobytes()
    assert np.array_equal(tg, tg2) and set(tg.tolist()) == {0, 1}


def _task_generator(core, seed=0):
    from mycroft_precise_b200.offline import Generator
    rs = np.random.RandomState(7)
    bgs = [np.clip(rs.randn(int(n)) * 600, -32768, 32767).astype(np.int16) for n in rs.randint(80000, 200000, 6)]
    wake = [train_task.clip(i, True)[:] for i in range(0, 40, 2)]
    other = [train_task.clip(i, False) for i in range(1, 40, 2)]
    return Generator(core, bgs, wake, other, chunk=2048, seed=seed)


def _state(fx, k=2):
    from mycroft_precise_b200.model_io import GruModel
    from mycroft_precise_b200.offline import TrainState
    return TrainState.from_models(fx.core, [GruModel.init(fx.core.feature_size, 20, s) for s in range(k)], list(range(k)))


@gpu
def test_training_is_deterministic_and_resumable(fx):
    from mycroft_precise_b200.offline import train_generated
    runs = []
    for _ in range(2):
        st = _state(fx)
        loss = train_generated(fx.core, st, _task_generator(fx.core), 3, steps_per_epoch=4, batch_size=50)
        runs.append((loss, st.weights.cpu().numpy()))
    assert runs[0][0].tobytes() == runs[1][0].tobytes() and runs[0][1].tobytes() == runs[1][1].tobytes()
    st = _state(fx)
    parts = [train_generated(fx.core, st, _task_generator(fx.core), 1, steps_per_epoch=4, batch_size=50) for _ in range(3)]
    assert np.concatenate(parts, 1).tobytes() == runs[0][0].tobytes()
    assert st.weights.cpu().numpy().tobytes() == runs[0][1].tobytes()


@gpu
def test_losses_match_the_float64_training_oracle(fx):
    from mycroft_precise_b200.offline import train_generated
    gen = _task_generator(fx.core, seed=5)
    x, tg, _, _ = gen.at(0, 200).run(gen.at(0, 200).plan(200))
    st = _state(fx, 1)
    F = fx.core.feature_size
    row, rms = st.weights.cpu().numpy()[0].astype(np.float64), np.zeros(ot.STRIDE)
    loss = train_generated(fx.core, st, gen, 1, steps_per_epoch=4, batch_size=50)
    want = ot.train_row(row, rms, F, 20, x.cpu().numpy().astype(np.float64), tg.astype(np.float64), np.arange(200), 0, 1,
                        batch_size=50)
    assert np.allclose(loss[0], want, rtol=1e-3), (loss[0], want)
    d = np.abs(st.weights.cpu().numpy()[0, :ot.row_size(F, 20)] - row[:ot.row_size(F, 20)])
    assert np.quantile(d, 0.99) < 1e-4, np.quantile(d, 0.99)


def _write(path, pcm, rate=16000):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with wave.open(path, 'wb') as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(rate)
        w.writeframes(np.ascontiguousarray(pcm, '<i2').tobytes())


def _read(path):
    with wave.open(path, 'rb') as w:
        return np.frombuffer(w.readframes(w.getnframes()), '<i2').astype(np.int16)


@gpu
def test_cli_writes_its_files_and_reaches_the_task(fx, tmp_path, capsys, monkeypatch):
    from mycroft_precise_b200 import train_generated as cli
    data, rnd = tmp_path / 'data', tmp_path / 'random'
    for i in range(40):
        _write(str(data / ('wake-word' if i % 2 == 0 else 'not-wake-word') / ('c%03d.wav' % i)), train_task.clip(i, i % 2 == 0))
    for i in range(6):
        _write(str(data / 'test' / ('wake-word' if i % 2 == 0 else 'not-wake-word') / ('t%d.wav' % i)), train_task.clip(500 + i, i % 2 == 0))
    rs = np.random.RandomState(2)
    for i in range(6):
        _write(str(rnd / ('bg%d.wav' % i)), np.clip(rs.randn(150000) * 600, -32768, 32767).astype(np.int16))
    model = str(tmp_path / 'm.npz')
    monkeypatch.chdir(tmp_path)
    cli.main([model, str(data), '-r', str(rnd), '-e', '2', '-t', '4', '-b', '50', '-p', '0.05'])
    text = capsys.readouterr().out
    assert '=== %s ===' % model in text and 'Epoch 2/2 - loss: ' in text and 'val_loss: ' in text
    assert os.path.isfile(model) and os.path.isfile(model + '.params')
    assert open(str(tmp_path / 'm.epoch')).read() == '2'
    saved = [os.path.join(r, n) for d in ('ww', 'nww') for r, _, ns in os.walk(str(tmp_path / 'debug' / d)) for n in ns]
    assert saved and all(_read(p).shape[0] == 24000 for p in saved)
    cli.main([model, str(data), '-r', str(rnd), '-e', '1', '-t', '4', '-b', '50'])        # resumes from the counter
    assert 'Epoch 3/3 - loss: ' in capsys.readouterr().out
    assert open(str(tmp_path / 'm.epoch')).read() == '3'


@gpu
def test_debug_wavs_are_the_stream_slices(fx, tmp_path):
    from mycroft_precise_b200.offline import _save_generated
    gen = _task_generator(fx.core, seed=1)
    plan = gen.plan(100)
    x, tg, audio, ends = gen.run(plan, out=True)
    _save_generated(gen, 0, plan, audio, ends, tg, 1.0, str(tmp_path))
    a = audio.cpu().numpy()
    j = 0
    for it, w0, w1 in plan:
        for c, t in it.windows[w0:w1]:
            name = os.path.join(str(tmp_path), 'ww' if tg[j] else 'nww', '%d - %d.wav' % (it.background, c))
            got = _read(name)
            e = int(ends[j])
            n = min(24000, (c + 1) * 2048)
            assert got.shape[0] == 24000 and not got[:24000 - n].any() and got[24000 - n:].tobytes() == a[e - n:e].tobytes()
            j += 1


@gpu
def test_chirp_task_reaches_held_out_accuracy(fx):
    m = fx.m
    core = m.PreciseB200()
    core.set_pool(1)
    gen = _task_generator(core)
    st = m.offline.TrainState.from_models(core, [m.GruModel.init(13, 20, 0)], [0])
    m.offline.train_generated(core, st, gen, 12, steps_per_epoch=10, batch_size=100)
    clips, targets = train_task.dataset(10000, train_task.N_TEST)
    core.pool_load(0, st.models()[0])
    acc = m.offline.test_pool(core, clips, targets, np.zeros(1, np.int32))[0].accuracy()
    core.close()
    print('held-out accuracy after generated training: %.3f' % acc)
    # 0.885 measured on an H100 (training is bit-deterministic).  The bar is below train_task's 0.9: the generated windows
    # are about 3 % positive, and a positive needs a wake-word run over 0.8 of the 1.5 s buffer, which the task's 0.75 ..
    # 1.25 s clips reach only where chunk_audio_pieces repeats a clip; the held-out clips are half wake words.
    assert acc >= 0.85
