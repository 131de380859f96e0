"""CPU-only: oracle/generated.py against the reference precise-train-generated's own run (tests/golden/generated_golden.npz,
made by make_generated_golden.py), and offline.Generator's host plan (segments, labels, keyed draws) against the literal
restatement."""
import os

import numpy as np

from oracle import generated as og
from oracle.listener import OracleListener
from oracle.params import OracleParams
from mycroft_precise_b200.offline import Generator, _LabelTail, _unit

HERE = os.path.dirname(os.path.abspath(__file__))
G = np.load(os.path.join(HERE, 'golden', 'generated_golden.npz'))

# |exact - 32767 literal| (int16 units) and the network-input difference of the int16 stream, measured below on the
# default front end: half a unit of rounding plus the literal form's float32 volume arithmetic, and the MFCC change that
# rounding makes (largest in the quiet frames of a silence over a quiet background: 0.063 measured here, over a background
# of RMS 40).
SAMPLE_BOUND = 0.52
MFCC_BOUND = 0.08


def _split(pcm, offsets):
    return [pcm[offsets[i]:offsets[i + 1]] for i in range(offsets.shape[0] - 1)]


def _golden_clips():
    return _split(G['bg_pcm'], G['bg_offsets']), _split(G['wake_pcm'], G['wake_offsets']), _split(G['other_pcm'], G['other_offsets'])


def test_literal_reproduces_every_golden_chunk_and_decision():
    bgs, wake, other = _golden_clips()
    lit = og.Literal(wake, other, G['draws'], int(G['chunk']), int(G['sample_rate']), int(G['buffer_samples']),
                     float(G['save_prob']))
    order = G['order']
    chunks, decisions = [], []
    for n in range(int(G['files'])):
        m, d = lit.file(bgs[order[n % len(order)]])
        chunks.append(m)
        decisions.append(d)
    assert np.array_equal(np.concatenate(chunks), G['chunks'])
    assert np.array_equal(np.concatenate(decisions), G['decisions'])
    assert lit.k == G['draws'].shape[0]                      # every draw, in the reference's order
    assert set(np.unique(G['decisions'])) == {-1, 0, 1}


def _keyed(gen, p, b):
    def draw(kind, k):
        if kind == 'volume':
            return _unit(gen.seed, p + 1, b, 0)
        if kind == 'piece':
            return _unit(gen.seed, p + 1, b, 1 + k)
        return 0.0                                            # save draws: never save
    return draw


def _walk(gen, wake, other, bgs, n_items):
    """(item, literal merged chunks, literal decisions, literal ww chunks, literal volume, pass, background) of the
    generator's next n_items items, the literal form run on the same keyed draws and state."""
    lit = og.Literal(wake, other, [], gen.chunk, gen.sample_rate, gen.buffer_samples)
    out = []
    for _ in range(n_items):
        p, b = gen.pass_, gen.order[gen.q]
        item = gen._next_item()
        lit.fn = _keyed(gen, p, b)
        m, d = lit.file(bgs[b])
        out.append((item, m, d, lit.ww, lit.volume, p, b))
    return out


def _segment_stream(item, clips, n_wake, volume):
    audio, label = [], []
    for c, a, m in item.segments:
        if c < 0:
            audio.append(np.zeros(m))
        else:
            audio.append(og._to_volume(og._load(clips[c]), volume).astype(np.float64)[a:a + m])
        label.append(np.full(m, 1.0 if 0 <= c < n_wake else 0.0))
    return np.concatenate(audio + [np.zeros(0)]), np.concatenate(label + [np.zeros(0)])


def test_segments_and_labels_are_the_literal_stream():
    bgs, wake, other = _golden_clips()
    for seed in (0, 1, 5):
        gen = Generator(None, bgs, wake, other, chunk=int(G['chunk']), seed=seed, sample_rate=int(G['sample_rate']),
                        buffer_samples=int(G['buffer_samples']))
        seen = set()
        for item, m, d, ww, vol, p, b in _walk(gen, wake, other, bgs, 14):
            assert item.length == m.shape[0] * gen.chunk
            audio, label = _segment_stream(item, wake + other, len(wake), vol)
            want = np.concatenate([w for w in ww], axis=1) if ww else np.zeros((2, 0))
            assert np.array_equal(audio, want[0]) and np.array_equal(label, want[1])
            assert item.windows == [(c, int(t)) for c, t in enumerate(d) if t >= 0]
            assert item.f == 0.4 + 0.5 * _unit(seed, p + 1, b, 0)
            seen.update(int(t) for t in d)
        assert seen == {-1, 0, 1}


def test_label_tail_is_max_run_length():
    rs = np.random.RandomState(3)
    B = 500
    tail, vals = _LabelTail(B), np.zeros(B)
    for _ in range(400):
        n, one = int(rs.randint(0, 300)), bool(rs.rand() < 0.5)
        tail.add(n, one)
        vals = np.concatenate([vals, np.full(n, float(one))])[-B:]
        frac = og.max_run(vals, 1) / B
        want = 1 if vals[-1] == 0 and frac > 0.8 else (0 if frac < 0.5 else -1)
        assert tail.decide(tail.end) == want


def test_key_layout():
    assert _unit(9, 1, 2, 3) == (0x138128F20561E1D9 >> 11) * 2.0 ** -53      # pb_train's key(9, 1, 2, 3)
    bgs, wake, other = _golden_clips()
    gen = Generator(None, bgs, wake, other, chunk=512, seed=9, sample_rate=4000, buffer_samples=3000)
    from mycroft_precise_b200.offline import _key
    assert gen.order == sorted(range(len(bgs)), key=lambda b: (_key(9, 0, b, 0), b))
    items = _walk(gen, wake, other, bgs, 6)
    for item, _, _, _, _, p, b in items:
        assert item.background == b
        if item.segments:                                                   # piece 0 draws u_1: a wake word if > 0.5
            assert (item.segments[0][0] < len(wake)) == (_unit(9, p + 1, b, 1) > 0.5)
    assert [x[5] for x in items] == [0, 0, 0, 0, 1, 1]                    # four backgrounds, cycled


def test_plan_resumes_and_cuts_items():
    bgs, wake, other = _golden_clips()
    kw = dict(chunk=512, seed=2, sample_rate=4000, buffer_samples=3000)
    whole = Generator(None, bgs, wake, other, **kw).plan(90)
    flat = lambda plan: [(it.background, it.f, c, t) for it, w0, w1 in plan for c, t in it.windows[w0:w1]]
    gen = Generator(None, bgs, wake, other, **kw)
    parts = [gen.plan(30) for _ in range(3)]
    assert sum((flat(p) for p in parts), []) == flat(whole)
    assert len(flat(whole)) == 90
    assert flat(Generator(None, bgs, wake, other, **kw).at(2, 30).plan(30)) == flat(parts[2])
    assert flat(gen.seek(30).plan(30)) == flat(parts[1])                  # replays from the start
    cut = [p for p in parts if p[0][1] > 0]
    assert cut, 'some epoch starts inside an item'


def _default_case():
    rs = np.random.RandomState(21)
    sig = lambda n, a: np.clip(np.round(rs.randn(n) * a), -32768, 32767).astype(np.int16)
    bgs = [sig(40000, 300), sig(30000, 2500), sig(52000, 40)]
    wake = [sig(12000, 4000), sig(16000, 3000)]
    other = [sig(9000, 2000), sig(20000, 800)]
    return bgs, wake, other


def test_exact_is_within_the_stated_bound_of_literal():
    bgs, wake, other = _default_case()
    pr = OracleParams()
    gen = Generator(None, bgs, wake, other, chunk=2048, seed=4, sample_rate=pr.sample_rate, buffer_samples=pr.buffer_samples)
    worst_s = worst_m = 0.0
    for item, m, d, ww, vol, p, b in _walk(gen, wake, other, bgs, 5):
        y = og.exact_item(bgs[b], wake + other, item.f, item.length, item.segments)
        lit = m.reshape(-1)
        worst_s = max(worst_s, float(np.max(np.abs(y - lit * 32767.0))))
        a, e = OracleListener(None, pr, 2048), OracleListener(None, pr, 2048)
        for k in range(m.shape[0]):
            va = a.update_vectors(m[k]).copy()
            ve = e.update_vectors(y[k * 2048:(k + 1) * 2048].astype(np.float64) / 32767.0)
            worst_m = max(worst_m, float(np.max(np.abs(va - ve))))
    print('max |exact - literal| = %.4f int16 units, max network-input difference %.4g' % (worst_s, worst_m))
    assert worst_s <= SAMPLE_BOUND
    assert worst_m <= MFCC_BOUND


def test_exact_rules_on_edge_cases():
    bg = np.full(8, 1000, np.int16)
    clip = np.asarray([0, 0, 0, 0], np.int16)                                # silent clip: gain 0
    assert og.exact_item(bg, [clip], 0.5, 8, [(0, 0, 4), (-1, 0, 4)]).tolist() == [200] * 8
    assert og.exact_item(np.zeros(8, np.int16), [np.full(4, 7, np.int16)], 0.9, 4, [(0, 0, 4)]).tolist() == [0] * 4
    loud = np.asarray([32767, 1, 1, 1], np.int16)
    got = og.exact_item(np.full(4, 32000, np.int16), [loud], 0.9, 4, [(0, 0, 4)])
    assert got[0] == 32767                                                     # saturates
    assert og.exact_item(bg, [clip], 0.4, 3, [(-1, 0, 1), (-1, 0, 0), (-1, 0, 5)]).tolist() == [160] * 3


def test_backgrounds_no_longer_than_a_chunk_are_refused():
    import pytest
    _, wake, other = _golden_clips()
    short = [np.zeros(512, np.int16), np.ones(100, np.int16)]
    with pytest.raises(ValueError, match='one chunk'):
        Generator(None, short, wake, other, chunk=512, sample_rate=4000, buffer_samples=3000)
    gen = Generator(None, short + [np.ones(513, np.int16)], wake, other, chunk=512, sample_rate=4000, buffer_samples=3000)
    assert len(gen.plan(5)) >= 1                                         # only the 513-sample background gives windows
