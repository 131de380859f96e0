"""CPU-only: oracle/noise.py against the reference precise-add-noise's own outputs (tests/golden/noise_golden.npz, made by
make_noise_golden.py), and the add_noise command's file order and output names."""
import os

import numpy as np

from oracle import noise as on

HERE = os.path.dirname(os.path.abspath(__file__))
G = np.load(os.path.join(HERE, 'golden', 'noise_golden.npz'))


def _split(pcm, offsets):
    return [pcm[offsets[i]:offsets[i + 1]] for i in range(offsets.shape[0] - 1)]


def _golden():
    clips = _split(G['clip_pcm'], G['clip_offsets'])
    outs = _split(G['out_pcm'], G['out_offsets'])
    M = int(G['inflation'])
    items = np.repeat(np.arange(len(clips)), M)
    return clips, outs, items, G['ratios']


def test_literal_reproduces_every_golden_sample():
    clips, outs, items, ratios = _golden()
    got, _ = on.literal(clips, G['noise_pcm'], items, ratios)
    assert len(got) == len(outs)
    for g, w in zip(got, outs):
        assert np.array_equal(g, w)


def test_exact_is_within_the_volume_ratio_bound_of_the_golden():
    clips, outs, items, ratios = _golden()
    noise = G['noise_pcm']
    got, _ = on.exact(clips, noise, items, ratios)
    starts, _ = on.positions([clips[i].shape[0] for i in items], noise.shape[0])
    worst = 0
    for g, w, i, p, r in zip(got, outs, items, starts, ratios):
        n = on.span(noise, p, clips[i].shape[0])
        v_exact, v_literal = on.volume_ratios(clips[i], n)
        delta = abs(v_exact - v_literal) / v_exact
        bound = 1 + np.abs(r * n.astype(np.float64) * v_exact) * delta
        diff = np.abs(g.astype(np.int64) - w.astype(np.int64))
        assert np.all(diff <= bound)
        worst = max(worst, int(diff.max()))
    assert worst <= 1


def test_cyclic_positions_match_the_golden():
    clips, _, items, _ = _golden()
    starts, end = on.positions([clips[i].shape[0] for i in items], G['noise_pcm'].shape[0])
    assert np.array_equal(starts, G['positions'])
    assert end == (int(G['positions'][-1]) + clips[items[-1]].shape[0]) % G['noise_pcm'].shape[0]


def test_ratios_are_the_seeded_stream():
    import random
    rnd = random.Random(int(G['seed']))
    u = np.asarray([rnd.random() for _ in range(G['draws'].shape[0])])
    assert np.array_equal(u, G['draws'])
    lo, hi = float(G['low']), float(G['high'])
    assert np.array_equal(lo + (hi - lo) * u, G['ratios'])


def test_cli_names_and_order_match_the_golden(tmp_path):
    from mycroft_precise_b200 import add_noise as cli
    folder = tmp_path / 'data'
    for rel in G['order']:
        p = folder / str(rel)
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_bytes(b'')
    files = cli.find_clips(str(folder))
    rel = [os.path.relpath(f, str(folder)) for f in files]
    assert sorted(rel) == sorted(str(r) for r in G['order'])
    groups = lambda names: [('test/' if n.startswith('test/') else '') + ('not-' if 'not-wake-word' in n else '') for n in names]
    assert groups(rel) == groups([str(r) for r in G['order']])                 # the reference's group order
    M = int(G['inflation'])
    names = [os.path.relpath(cli.output_name(str(folder), os.path.join(str(folder), str(r)), n, str(tmp_path / 'out')),
                             str(tmp_path / 'out')) for r in G['order'] for n in range(M)]
    assert names == [str(n) for n in G['out_names']]


def test_exact_rules_on_edge_cases():
    x = np.asarray([1000, -2000, 3000], np.int16)
    assert np.array_equal(on.exact_one(x, np.zeros(3, np.int16), 0.5), (x // 2).astype(np.int16))     # silent span: no noise
    assert np.array_equal(on.exact_one(np.zeros(3, np.int16), np.asarray([5, -5, 5], np.int16), 0.7), np.zeros(3, np.int16))
    four = lambda v: np.full(4, v, np.int16)
    spike = np.asarray([1, 0, 0, 0], np.int16)                   # all the noise's energy in one sample: gain 2 |x| r
    assert on.exact_one(four(20000), spike, 0.75).tolist() == [32767, 5000, 5000, 5000]           # saturates
    assert on.exact_one(four(-20000), -spike, 0.75).tolist() == [-32768, -5000, -5000, -5000]
    assert on.span(np.arange(3, dtype=np.int16), 2, 7).tolist() == [2, 0, 1, 2, 0, 1, 2]
