"""Labelled-clip statistics without a device: the numpy restatement of pb_score_dataset's integer statistics
(oracle/dataset.py) and offline.DatasetStats on top of them reproduce every number the reference's Stats gives
(tests/golden/stats_golden.npz, generated from precise/stats.py, calc_threshold.py and ThresholdDecoder.encode), and the
command-line tool finds the clips the reference's folder walk finds."""
import os
import wave

import numpy as np
import pytest

from oracle import dataset as od


@pytest.fixture(scope='module')
def g(golden_dir):
    return np.load(os.path.join(golden_dir, 'stats_golden.npz'))


def _stats(g, sel=slice(None)):
    from mycroft_precise_b200.offline import DatasetStats
    return DatasetStats(g['thresholds'], *od.dataset_stats(g['outputs'][sel], g['targets'][sel], g['thresholds']))


def test_golden_has_the_edge_cases(g):
    out, thr = g['outputs'], g['thresholds']
    assert (out == 0).any() and (out == 1).any() and np.isin(thr, out).sum() >= 5 and thr.dtype == np.float32


def test_counts_and_rates_equal_the_reference(g):
    st = _stats(g)
    assert (int(st.count[1]), int(st.count[0]), len(st)) == (int(g['num_positives']), int(g['num_negatives']), len(g['outputs']))
    for j, t in enumerate(g['thresholds']):
        got = [st.true_pos(t), st.true_neg(t), st.false_pos(t), st.false_neg(t), st.num_correct(t)]
        assert got == g['metrics'][j].tolist(), (j, t)
        assert st.num_incorrect(t) == len(st) - g['metrics'][j][4]
        assert [st.false_positives(t), st.false_negatives(t), st.accuracy(t)] == g['rates'][j].tolist()
        assert st.counts_str(t) == str(g['counts_str'][j])
        assert st.summary_str(t) == str(g['summary_str'][j])
    # where an output equals the threshold, > and >= really differ
    assert any(st._above(l, t, True) != st._above(l, t, False) for t in g['thresholds'] for l in (0, 1))


def test_python_float_thresholds_and_unknown_ones(g):
    st = _stats(g)
    assert st.true_pos(0.5) == st.true_pos(np.float32(0.5)) and st.false_pos(0.1) == int(g['metrics'][list(g['thresholds']).index(np.float32(0.1))][2])
    with pytest.raises(KeyError):
        st.true_pos(0.3)
    with pytest.raises(KeyError):
        st.num_correct(2.0)


def test_histogram_bins(g):
    thr = np.float32([0.25, 0.5])
    x = np.float32([0.0, 0.25, 0.3, 0.5, 0.5, 0.7, 1.0, np.nan])
    count, hist, fit = od.dataset_stats(x, [1] * 8, thr)
    assert count.tolist() == [0, 8] and hist[0].sum() == 0
    assert hist[1].tolist() == [2, 1, 1, 2, 2]                  # NaN lands in bin 0
    assert fit[1][0] == 5 and fit[0].tolist() == [0, 0, 0]     # 0, 1 and NaN are no data for the fit


def test_fit_matches_calc_threshold(g):
    from mycroft_precise_b200.offline import calc_threshold
    st = _stats(g)
    mu, std = calc_threshold(st)
    ref_mu, ref_std = g['fit']                                 # the reference's own statements, float32 inside
    assert abs(mu - ref_mu) < 1e-6 and abs(std - ref_std) < 1e-6
    o_mu, o_std = od.calc_threshold(g['outputs'], g['targets'])
    # float64 throughout: 1 / x - 1 is not rounded to float32, which moves v of the outputs next to 1 in the 5th digit
    assert abs(mu - o_mu) < 1e-4 and abs(std - o_std) < 1e-4
    assert calc_threshold(st, smoothing=1.0)[1] == pytest.approx(std / 1.2, rel=1e-12)
    none = _stats(g, slice(0, 4))                              # outputs 0, 1, 0, 1 only
    assert calc_threshold(none) is None and od.calc_threshold(g['outputs'][:4], g['targets'][:4]) is None


def test_statistics_add(g):
    a, b = _stats(g, slice(0, 2500)), _stats(g, slice(2500, None))
    s, whole = a + b, _stats(g)
    assert np.array_equal(s.count, whole.count) and np.array_equal(s.hist, whole.hist) and np.array_equal(s.fit, whole.fit)
    from mycroft_precise_b200.offline import DatasetStats
    other = DatasetStats(np.float32([0.5]), *od.dataset_stats(g['outputs'], g['targets'], [0.5]))
    with pytest.raises(ValueError):
        a + other


def test_graph_thresholds_and_roc(g):
    from golden.cases import DECODER_CASES
    from mycroft_precise_b200 import ListenerParams
    from mycroft_precise_b200.core import threshold_encode
    from mycroft_precise_b200.offline import DatasetStats, graph_thresholds, roc
    seen = 0
    for i, (cfg, center) in enumerate(DECODER_CASES):
        if 'graph_%d' % i not in g:
            continue
        seen += 1
        want = g['graph_%d' % i]
        assert np.array_equal(threshold_encode(cfg, center, np.linspace(0.0, 1.0, 100)[1:-1]), want)
        thr = graph_thresholds(ListenerParams(threshold_config=cfg, threshold_center=center))
        assert thr.dtype == np.float32 and np.all(np.diff(thr) > 0) and np.array_equal(thr, np.unique(want.astype(np.float32)))
    assert seen >= 4
    thr = graph_thresholds(ListenerParams())
    st = DatasetStats(thr, *od.dataset_stats(g['outputs'], g['targets'], thr))
    fp, fn = roc(st)
    out, pos = g['outputs'], g['targets'] > 0.5
    assert np.array_equal(fp, [(out[~pos] > t).sum() / (~pos).sum() for t in thr])
    assert np.array_equal(fn, [(~(out[pos] > t)).sum() / pos.sum() for t in thr])
    assert np.all(np.diff(fp) <= 0) and np.all(np.diff(fn) >= 0)


def _wav(path, n, rate=16000):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with wave.open(path, 'wb') as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(rate)
        w.writeframes((np.arange(n) % 100).astype('<i2').tobytes())


def test_folder_walk(tmp_path):
    from mycroft_precise_b200.test import load_folder
    root = str(tmp_path)
    _wav(os.path.join(root, 'wake-word', 'a.wav'), 100)
    _wav(os.path.join(root, 'not-wake-word', 'b.wav'), 200)
    _wav(os.path.join(root, 'test', 'wake-word', 'c.wav'), 300)
    _wav(os.path.join(root, 'test', 'wake-word', 'deep', 'er', 'd.wav'), 400)
    _wav(os.path.join(root, 'test', 'wake-word', 'empty.wav'), 0)
    _wav(os.path.join(root, 'test', 'not-wake-word', 'e.wav'), 500)
    open(os.path.join(root, 'test', 'not-wake-word', 'notes.txt'), 'w').write('x')
    open(os.path.join(root, 'test', 'not-wake-word', 'broken.wav'), 'w').write('x')
    files, clips, targets = load_folder(root, use_train=False)
    assert sorted(os.path.basename(f) for f in files) == ['c.wav', 'd.wav', 'e.wav']
    assert {os.path.basename(f): (len(c), int(t)) for f, c, t in zip(files, clips, targets)} == \
        {'c.wav': (300, 1), 'd.wav': (400, 1), 'e.wav': (500, 0)}
    assert targets.tolist() == [1, 1, 0] and targets.dtype == np.uint8 and all(c.dtype == np.int16 for c in clips)
    files, clips, targets = load_folder(root, use_train=True)
    assert [os.path.basename(f) for f in files] == ['a.wav', 'b.wav'] and targets.tolist() == [1, 0]
    with pytest.raises(ValueError):
        _wav(os.path.join(root, 'test', 'wake-word', 'slow.wav'), 100, rate=8000)
        load_folder(root, use_train=False)
