"""Noise augmentation on the device (pb_add_noise; PreciseB200.add_noise, offline.NoiseSource / add_noise / vectorize_noisy /
Augment, train(augment=...), python -m mycroft_precise_b200.add_noise and train --noise-folder) against oracle/noise.py's
exact restatement and the existing vectorize and training paths.  -m gpu."""
import ctypes as C
import os
import sys
import wave

import numpy as np
import pytest

from oracle import noise as on
from oracle import train as ot

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import train_task  # noqa: E402

gpu = pytest.mark.gpu
F, T = 13, 29


def _sig(n, seed, sigma=3000):
    rs = np.random.RandomState(seed)
    return np.clip(np.round(rs.randn(n) * sigma), -32768, 32767).astype(np.int16)


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


class Fixture:
    def __init__(self):
        import torch
        import mycroft_precise_b200 as m
        self.m, self.torch = m, torch
        self.core = m.PreciseB200()

    def dev(self, a):
        return self.torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.fixture(scope='module')
def fx():
    pytest.importorskip('torch')
    f = Fixture()
    yield f
    f.core.close()


def _packed(clips, lead=3):
    """Clips back to back after `lead` samples (odd offsets): (pcm, offsets), recording 0 the lead and r + 1 clip r."""
    parts = [_sig(lead, 999)] + list(clips)
    offsets = np.concatenate([[0], np.cumsum([len(c) for c in parts])]).astype(np.int64)
    return np.concatenate(parts), offsets


def _split(pcm, lens):
    o = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    return [pcm[o[i]:o[i + 1]] for i in range(len(lens))]


def _case():
    lens = [1, 2, 7, 511, 1600, 4097, 24000, 24001, 30001, 100000, 333]
    clips = [_sig(n, 10 + i, 1500 + 300 * i) for i, n in enumerate(lens)]
    clips[3][:] = 0                                                        # a silent clip
    clips.append(np.full(64, 20000, np.int16))                             # saturates against the spike below
    noise = _sig(7001, 77, 2500)
    noise[100:164] = 0                                                     # a silent span
    noise[5000:5064] = 0
    noise[5000] = 1
    return clips, noise


# ---- 1. mixing ----------------------------------------------------------------------------------------------------------------

@gpu
def test_add_noise_is_the_exact_oracle(fx):
    clips, noise = _case()
    pcm, offsets = _packed(clips)
    n = len(clips)
    rs = np.random.RandomState(5)
    # every clip once, then repeats; ratios 0 and 1 among random ones; spans wrapping once (30001, 100000 > 7001) and many
    # times.  Below: the silent span (the 7-sample clip from position 100) and the spike (the last clip from 5000)
    items = np.concatenate([np.arange(1, n + 1), [5, 5, 9, 1], [4, n]]).astype(np.int32)
    ratios = rs.rand(items.size)
    ratios[[0, 3]] = 0.0
    ratios[[1, 7]] = 1.0
    ratios[-1] = 0.75
    host_clips = [pcm[offsets[r]:offsets[r + 1]] for r in range(n + 1)]
    lens = [host_clips[i].shape[0] for i in items]
    for pos in (0, 4321, 7000):
        want, end = on.exact(host_clips, noise, items, ratios, pos)
        out, _ = fx.core.add_noise(fx.dev(pcm), offsets, fx.dev(noise), items, ratios, pos)
        got = _split(out.cpu().numpy(), lens)
        for j, (g, w) in enumerate(zip(got, want)):
            assert _same(g, w), (pos, j, int(np.abs(g.astype(int) - w).max()))
    # the silent span and the saturating spike, each at its own position
    for item, pos, r in ((3, 100, 0.5), (n, 5000, 0.75)):
        want, _ = on.exact(host_clips, noise, [item], [r], pos)
        out, _ = fx.core.add_noise(fx.dev(pcm), offsets, fx.dev(noise), [item], [r], pos)
        assert _same(out.cpu().numpy(), want[0])
    w = on.exact(host_clips, noise, [n], [0.75], 5000)[0][0]
    assert w[0] == 32767
    w = on.exact(host_clips, noise, [3], [0.5], 100)[0][0]                  # the silent span adds nothing
    assert np.array_equal(w, np.trunc(0.5 * host_clips[3].astype(np.float64)).astype(np.int16))


@gpu
def test_split_calls_equal_one_call(fx):
    clips, noise = _case()
    pcm, offsets = _packed(clips)
    items = np.arange(1, len(clips) + 1, dtype=np.int32)
    ratios = np.random.RandomState(8).rand(items.size)
    dpcm, dnoise = fx.dev(pcm), fx.dev(noise)
    one, _ = fx.core.add_noise(dpcm, offsets, dnoise, items, ratios, 17)
    parts, pos = [], 17
    for a, b in ((0, 4), (4, 5), (5, len(items))):
        o, _ = fx.core.add_noise(dpcm, offsets, dnoise, items[a:b], ratios[a:b], pos)
        parts.append(o.cpu().numpy())
        pos = (pos + int(np.diff(offsets)[items[a:b]].sum())) % noise.shape[0]
    assert _same(np.concatenate(parts), one.cpu().numpy())
    # offline: a NoiseSource carries the position; the clips split into several library calls give the same result
    m = fx.m
    host = [pcm[offsets[r]:offsets[r + 1]] for r in range(1, len(clips) + 1)]
    src = m.offline.NoiseSource(fx.core, [noise[:3000], np.zeros(0, np.int16), noise[3000:]], pos=17)
    a, ao = m.offline.add_noise(fx.core, host, src, ratios)
    assert _same(a.cpu().numpy(), one.cpu().numpy()) and src.pos == pos
    old = m.offline.CORPUS_CALL_SAMPLES
    try:
        m.offline.CORPUS_CALL_SAMPLES = 40000
        src.pos = 17
        b, bo = m.offline.add_noise(fx.core, host, src, ratios)
        assert src.pos == pos
        src.pos = 17
        vb = m.offline.vectorize_noisy(fx.core, host[:3] + host[4:], src, ratios[:10], np.arange(10))
    finally:
        m.offline.CORPUS_CALL_SAMPLES = old
    src.pos = 17
    va = m.offline.vectorize_noisy(fx.core, host[:3] + host[4:], src, ratios[:10], np.arange(10))
    assert _same(b.cpu().numpy(), a.cpu().numpy()) and np.array_equal(ao, bo)
    assert _same(va.cpu().numpy(), vb.cpu().numpy())


# ---- 2. vectorizing -----------------------------------------------------------------------------------------------------------

def _aligned(clips, ms):
    """The clips' last ms samples, each starting at a multiple of 8 (1..7-sample filler entries between): (pcm, offsets,
    entry of each clip)."""
    parts, entry, pos = [], [], 0
    for c in clips:
        c = c[-ms:]
        if pos % 8:
            parts.append(np.ones(8 - pos % 8, np.int16))
            pos += 8 - pos % 8
        entry.append(len(parts))
        parts.append(c)
        pos += c.shape[0]
    offsets = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int64)
    return np.concatenate(parts), offsets, np.asarray(entry)


@gpu
@pytest.mark.parametrize('generic', [False, True])
def test_inputs_are_vectorize_clips_of_the_mixed_clips(fx, generic):
    clips, noise = _case()
    clips = clips[1:3] + clips[4:]                                           # none empty
    pcm, offsets = _packed(clips)
    items = np.concatenate([np.arange(1, len(clips) + 1), [2, 2, 6]]).astype(np.int32)
    ratios = np.random.RandomState(9).rand(items.size)
    ms = fx.core.params.max_samples
    lens = np.diff(offsets)[items]
    fx.core.force_generic(generic)
    try:
        out, x = fx.core.add_noise(fx.dev(pcm), offsets, fx.dev(noise), items, ratios, 555, inputs=True)
        none, x2 = fx.core.add_noise(fx.dev(pcm), offsets, fx.dev(noise), items, ratios, 555, out=False, inputs=True)
        mixed = _split(out.cpu().numpy(), lens)
        apcm, aoff, entry = _aligned(mixed, ms)
        want = fx.core.vectorize_clips(fx.dev(apcm), aoff).cpu().numpy()[entry]
        if generic:                                                          # offline.vectorize_clips packs its own way
            src = fx.m.offline.NoiseSource(fx.core, [noise], 555)
            host = [pcm[offsets[r]:offsets[r + 1]] for r in range(len(clips) + 1)]
            v = fx.m.offline.vectorize_noisy(fx.core, host, src, ratios, items)
            src.pos = 555
            o, _ = fx.m.offline.add_noise(fx.core, host, src, ratios, items)
            w2 = fx.m.offline.vectorize_clips(fx.core, _split(o.cpu().numpy(), lens))
            assert _same(v.cpu().numpy(), w2.cpu().numpy())
    finally:
        fx.core.force_generic(False)
    assert none is None
    assert _same(x.cpu().numpy(), want) and _same(x2.cpu().numpy(), want)


# ---- 3. refusals --------------------------------------------------------------------------------------------------------------

@gpu
def test_refusals_change_no_buffer(fx):
    core, torch = fx.core, fx.torch
    lib = core.lib
    clips = [_sig(3000, 1), np.zeros(0, np.int16), _sig(500, 2)]
    pcm, offsets = _packed(clips)
    dpcm, dnoise = fx.dev(pcm), fx.dev(_sig(999, 3))
    out = torch.full((10000,), 1234, dtype=torch.int16, device='cuda')
    inp = torch.full((4, T, F), 7.0, dtype=torch.float32, device='cuda')
    P = lambda t: None if t is None else C.c_void_p(t.data_ptr())

    def call(items=(1, 3), ratios=(0.5, 0.25), n_noise=999, pos=0, divisor=32767, ms=24000, d_out=out, d_in=inp, noise=dnoise,
             n_rec=4):
        it = np.asarray(items, np.int32)
        r = np.asarray(ratios, np.float64)
        return lib.pb_add_noise(core._h, P(dpcm), offsets.ctypes.data_as(C.c_void_p), n_rec, P(noise), n_noise,
                                it.ctypes.data_as(C.c_void_p), r.ctypes.data_as(C.c_void_p), it.size, pos, divisor, ms,
                                P(d_out), P(d_in), None)
    bad = [dict(n_noise=0), dict(pos=-1), dict(pos=999), dict(items=(1, 4)), dict(items=(-1, 1)), dict(ratios=(0.5, np.nan)),
           dict(ratios=(0.5, 1.0000001)), dict(ratios=(-0.1, 0.5)), dict(d_out=None, d_in=None), dict(items=(1, 2)),
           dict(divisor=1000), dict(ms=0), dict(noise=None), dict(n_rec=-1)]
    for kw in bad:
        assert call(**kw) == -1, kw
        torch.cuda.synchronize()
        assert bool((out == 1234).all()) and bool((inp == 7.0).all()), kw
    # an empty item is fine with d_out alone
    assert call(items=(1, 2, 3), ratios=(0.5, 0.5, 0.5), d_in=None) == 0
    torch.cuda.synchronize()
    assert bool((out[3500:] == 1234).all()) and not bool((out[:3500] == 1234).all())
    # d_inputs on a front end outside the fused family
    core2 = fx.m.PreciseB200(fx.m.ListenerParams(use_delta=True))
    assert lib.pb_add_noise(core2._h, P(dpcm), offsets.ctypes.data_as(C.c_void_p), 4, P(dnoise), 999,
                            np.asarray([1], np.int32).ctypes.data_as(C.c_void_p),
                            np.asarray([0.5]).ctypes.data_as(C.c_void_p), 1, 0, 32767, 24000, None, P(inp), None) == -2
    core2.close()


# ---- 4. the command -----------------------------------------------------------------------------------------------------------

def _write(path, pcm):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with wave.open(path, 'wb') as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(16000)
        w.writeframes(np.ascontiguousarray(pcm, '<i2').tobytes())


def _read(path):
    with wave.open(path, 'rb') as w:
        assert (w.getnchannels(), w.getsampwidth(), w.getframerate()) == (1, 2, 16000)
        return np.frombuffer(w.readframes(w.getnframes()), '<i2').astype(np.int16)


@gpu
def test_cli_writes_what_the_oracle_predicts(tmp_path, capsys):
    import random
    from mycroft_precise_b200 import add_noise as cli
    data, nz, out = str(tmp_path / 'data'), str(tmp_path / 'noise'), str(tmp_path / 'out')
    clips = {'wake-word/b.wav': _sig(4000, 1), 'wake-word/a.wav': _sig(16001, 2), 'wake-word/x/c.wav': _sig(7, 3),
             'not-wake-word/z.wav': _sig(2222, 4), 'test/wake-word/t.wav': _sig(30000, 5), 'test/not-wake-word/u.wav': _sig(99, 6)}
    for rel, a in clips.items():
        _write(os.path.join(data, rel), a)
    noises = {'b.wav': _sig(3000, 7), 'a.wav': _sig(1234, 8), 'c.wav': np.zeros(0, np.int16)}
    for rel, a in noises.items():
        _write(os.path.join(nz, rel), a)
    cli.main([data, nz, out, '-if', '3', '-nl', '0.1', '-nh', '0.7', '--seed', '4'])
    order = ['wake-word/a.wav', 'wake-word/b.wav', 'wake-word/x/c.wav', 'not-wake-word/z.wav', 'test/wake-word/t.wav',
             'test/not-wake-word/u.wav']
    rnd = random.Random(4)
    ratios = [0.1 + 0.6 * rnd.random() for _ in range(3 * len(order))]
    noise = on.corpus([noises[k] for k in sorted(noises)])
    want, _ = on.exact([clips[k] for k in order], noise, np.repeat(np.arange(len(order)), 3), ratios)
    names = []
    for i, rel in enumerate(order):
        for n in range(3):
            base, ext = os.path.splitext(rel)
            names.append(rel if n == 0 else '%s.%d%s' % (base, n, ext))
    written = sorted(os.path.relpath(os.path.join(r, f), out) for r, _, fs in os.walk(out) for f in fs)
    assert written == sorted(names)
    for name, w in zip(names, want):
        assert _same(_read(os.path.join(out, name)), w), name
    # the 100th pass over the noise warns once; an empty corpus exits instead of hanging
    for rel in noises:
        os.remove(os.path.join(nz, rel))
    _write(os.path.join(nz, 'tiny.wav'), _sig(5, 9))
    capsys.readouterr()
    cli.main([data, nz, str(tmp_path / 'out2')])
    assert capsys.readouterr().out.count(cli.REPEAT_WARNING) == 1
    os.remove(os.path.join(nz, 'tiny.wav'))
    _write(os.path.join(nz, 'empty.wav'), np.zeros(0, np.int16))
    with pytest.raises(SystemExit):
        cli.main([data, nz, str(tmp_path / 'out3')])


# ---- 5. training --------------------------------------------------------------------------------------------------------------

def _task(n):
    clips, tg = train_task.dataset(0, n)
    return clips, tg


@gpu
def test_train_augment_is_the_hand_written_loop(fx):
    m, core, torch = fx.m, fx.core, fx.torch
    clips, tg = _task(24)
    noise = [_sig(50000, 31, 1000), _sig(20000, 32, 3000)]
    M, E = 2, 3
    init = [m.GruModel.init(F, 20, 0), m.GruModel.init(F, 8, 1)]
    rows = np.asarray([0, 0, 1, 1, 1], np.int32)
    recs = np.asarray([0, 5, 5, 7, 23], np.int64)

    def fit(epochs, state=None, pairs=False, pos=123):
        state = state or m.offline.TrainState.from_models(core, init, [3, 4])
        aug = m.offline.Augment(m.offline.NoiseSource(core, noise, pos), M, 0.05, 0.5, seed=9)
        kw = dict(rows=rows, recs=recs) if pairs else {}
        loss = m.offline.train(core, state, clips, tg, epochs=epochs, batch_size=7, augment=aug, **kw)
        return state, loss

    a, la = fit(E)
    b, lb = fit(E)
    assert _same(a.weights.cpu().numpy(), b.weights.cpu().numpy()) and _same(la, lb)
    c, lc = fit(1)
    for _ in range(E - 1):
        c, l1 = fit(1, c)
        lc = np.concatenate([lc, l1], 1)
    assert _same(a.weights.cpu().numpy(), c.weights.cpu().numpy()) and _same(la, lc)
    # the hand-written loop: vectorize_noisy at the epoch's position and ratios, then pb_train with epochs = 1
    st = m.offline.TrainState.from_models(core, init, [3, 4])
    clean = m.offline.vectorize_clips(core, clips)
    total = sum(len(c) for c in clips)
    src = m.offline.NoiseSource(core, noise, 123)
    N = len(src)
    items = np.repeat(np.arange(len(clips)), M)
    losses = []
    for e in range(E):
        u = np.asarray([(ot.key(9, e, i, 0) >> 11) * 2.0 ** -53 for i in range(items.size)])
        src.pos = (123 + e * M * total) % N
        noisy = m.offline.vectorize_noisy(core, clips, src, 0.05 + 0.45 * u, items).view(len(clips), M, T, F)
        x = torch.cat([clean[:, None], noisy], 1).reshape(-1, T, F).contiguous()
        losses.append(core.train(x, np.repeat(tg, M + 1), st.rows, st.weights, st.rms, epochs=1, epoch0=e, batch_size=7))
    assert _same(st.weights.cpu().numpy(), a.weights.cpu().numpy())
    assert _same(torch.cat(losses, 1).cpu().numpy(), la)
    # pairs expand to each clip's clean and noisy entries
    p, lp = fit(1, pairs=True)
    st = m.offline.TrainState.from_models(core, init, [3, 4])
    u = np.asarray([(ot.key(9, 0, i, 0) >> 11) * 2.0 ** -53 for i in range(items.size)])
    src.pos = 123
    noisy = m.offline.vectorize_noisy(core, clips, src, 0.05 + 0.45 * u, items).view(len(clips), M, T, F)
    x = torch.cat([clean[:, None], noisy], 1).reshape(-1, T, F).contiguous()
    r2 = np.repeat(rows, M + 1)
    c2 = np.concatenate([[3 * r + j for j in range(3)] for r in recs]).astype(np.int32)
    l2 = core.train(x, np.repeat(tg, M + 1), st.rows, st.weights, st.rms, epochs=1, epoch0=0, batch_size=7, rows_of=r2, recs=c2)
    assert _same(st.weights.cpu().numpy(), p.weights.cpu().numpy()) and _same(l2.cpu().numpy(), lp)


@gpu
def test_train_augment_losses_match_the_float64_oracle(fx):
    m, core = fx.m, fx.core
    clips, tg = _task(16)
    noise = [_sig(40000, 41, 1500)]
    M = 1
    init = m.GruModel.init(F, 20, 0)
    state = m.offline.TrainState.from_models(core, [init], [5])
    w0 = state.weights.cpu().numpy()[0].astype(np.float64)
    aug = m.offline.Augment(m.offline.NoiseSource(core, noise, 0), M, 0.0, 0.4, seed=2)
    loss = m.offline.train(core, state, clips, tg, epochs=1, batch_size=8, augment=aug)
    # the oracle-mixed clips, vectorized on the device (the inputs' own accuracy is test_gpu_train's)
    u = np.asarray([(ot.key(2, 0, i, 0) >> 11) * 2.0 ** -53 for i in range(len(clips))])
    mixed, _ = on.exact(clips, on.corpus(noise), np.arange(len(clips)), 0.4 * u, 0)
    x = m.offline.vectorize_clips(core, [c for pair in zip(clips, mixed) for c in pair]).cpu().numpy().astype(np.float64)
    row, rms = w0.copy(), np.zeros(ot.STRIDE)
    want = ot.train_row(row, rms, F, 20, x, np.repeat(tg, 2).astype(np.float64), np.arange(2 * len(clips)), 5, 1, batch_size=8)
    assert np.allclose(loss[0], want, rtol=1e-3), (loss[0], want)
    d = np.abs(state.weights.cpu().numpy()[0, :ot.row_size(F, 20)] - row[:ot.row_size(F, 20)])
    assert np.quantile(d, 0.99) < 1e-4 and d.max() < 12 * 2 * 0.001 / np.sqrt(0.1), (np.quantile(d, 0.99), d.max())


@gpu
def test_augmented_training_still_learns_the_task(fx):
    m = fx.m
    clips, tg = train_task.dataset(0, train_task.N_TRAIN)
    t_clips, t_tg = train_task.dataset(10000, train_task.N_TEST)
    core = m.PreciseB200()
    core.set_pool(1)
    init = m.GruModel.init(13, 20, 0)
    state = m.offline.TrainState.from_models(core, [init], [0])
    noise = [_sig(160000, 51, 800)]
    aug = m.offline.Augment(m.offline.NoiseSource(core, noise), 1, 0.0, 0.4, seed=0)
    loss, val = m.offline.train(core, state, clips, tg, epochs=train_task.EPOCHS, batch_size=train_task.BATCH,
                                validation=(m.offline.vectorize_clips(core, t_clips), t_tg), augment=aug)
    assert loss.shape == val.shape == (1, train_task.EPOCHS)
    core.pool_load(0, state.models()[0])
    acc = m.offline.test_pool(core, t_clips, t_tg, np.zeros(1, np.int32))[0].accuracy()
    assert acc >= train_task.MIN_ACCURACY, acc
    core.close()


@gpu
def test_train_command_with_noise_folder(tmp_path):
    from mycroft_precise_b200 import train as cli
    data, nz = str(tmp_path / 'data'), str(tmp_path / 'noise')
    clips, tg = _task(12)
    for i, (c, t) in enumerate(zip(clips, tg)):
        _write(os.path.join(data, 'wake-word' if t else 'not-wake-word', '%02d.wav' % i), c)
    _write(os.path.join(nz, 'n.wav'), _sig(30000, 61, 900))
    model = str(tmp_path / 'm.npz')
    loss = cli.main([model, data, '-e', '2', '-b', '8', '--noise-folder', nz, '-if', '2'])
    assert loss.shape == (1, 2) and np.all(np.isfinite(loss))
