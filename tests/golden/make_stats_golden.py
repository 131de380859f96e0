#!/usr/bin/env python3
"""Generate stats_golden.npz from the REAL reference code (see make_golden.py for the other fixtures):

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_stats_golden.py /path/to/mycroft-precise

Taken from the reference, unmodified:
  * precise.stats.Stats (pure numpy)                      -> every count, rate and format string, per threshold
  * precise/scripts/calc_threshold.py, the statements from ``save_spots =`` to ``pos_std =``, compiled from the checkout's
    file at generation time (the script itself imports a command-line package this image lacks)  -> fit_mu, fit_std
  * precise.threshold_decoder.ThresholdDecoder.encode    -> precise-graph's thresholds (graph.py:147-148)
The inputs are seeded float32 "network outputs", among them outputs equal to a threshold, 0.0 and 1.0.
"""
import os
import sys
import textwrap
import types
from math import sqrt

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.dont_write_bytecode = True
REF = os.path.abspath(sys.argv[1])
sys.path.insert(0, REF)
sys.path.insert(0, HERE)

from cases import DECODER_CASES                                    # noqa: E402
from precise.stats import Stats                                    # noqa: E402
from precise.threshold_decoder import ThresholdDecoder             # noqa: E402


def reference_fit():
    """calc_threshold.py's fit as a function of (stats, args): its own statements, wrapped."""
    lines = open(os.path.join(REF, 'precise', 'scripts', 'calc_threshold.py')).read().splitlines()
    a = next(i for i, l in enumerate(lines) if 'save_spots =' in l)
    b = next(i for i, l in enumerate(lines) if 'pos_std =' in l)
    body = textwrap.dedent('\n'.join(lines[a:b + 1]))
    src = 'def fit(stats, args):\n' + textwrap.indent(body, '    ') + '\n    return pos_mu, pos_std\n'
    env = {'np': np, 'sqrt': sqrt}
    exec(compile(src, 'calc_threshold.py', 'exec'), env)
    return env['fit']


def main():
    rs = np.random.RandomState(23)
    n = 6000
    targets = (rs.rand(n) < 0.4).astype(np.float64)
    logits = np.where(targets > 0.5, rs.randn(n) * 4 + 6, rs.randn(n) * 3 - 5).astype(np.float32)
    outputs = (1.0 / (1.0 + np.exp(-logits))).astype(np.float32)
    outputs[:8] = np.float32([0.0, 1.0, 0.0, 1.0, 0.5, 0.5, 0.9, 0.1])
    targets[:8] = [0, 1, 1, 0, 1, 0, 1, 0]
    thresholds = np.unique(np.concatenate([np.float32([0.5, 0.1, 0.9, 0.25, 0.999]), outputs[[10, 99, 1234, 4000]]]))
    stats = Stats(outputs, targets, ['%d.wav' % i for i in range(n)])
    out = dict(outputs=outputs, targets=targets, thresholds=thresholds,
               num_positives=np.int64(stats.num_positives), num_negatives=np.int64(stats.num_negatives))
    rows, counts, summaries = [], [], []
    for t in thresholds:
        t = float(t)
        d = stats.to_dict(t)
        rows.append([d['true_pos'], d['true_neg'], d['false_pos'], d['false_neg'], int(stats.num_correct(t))])
        counts.append(stats.counts_str(t))
        summaries.append(stats.summary_str(t))
    out['metrics'] = np.asarray(rows, np.int64)                 # true_pos, true_neg, false_pos, false_neg, num_correct
    out['rates'] = np.asarray([[stats.false_positives(float(t)), stats.false_negatives(float(t)), stats.accuracy(float(t))]
                               for t in thresholds], np.float64)
    out['counts_str'] = np.asarray(counts)
    out['summary_str'] = np.asarray(summaries)
    out['miss_files'] = np.asarray(stats.calc_filenames(False, True, 0.5) + stats.calc_filenames(False, False, 0.5))
    mu, std = reference_fit()(Stats(outputs, targets, []), types.SimpleNamespace(smoothing=1.2))
    out['fit'] = np.asarray([mu, std], np.float64)
    for i, (cfg, center) in enumerate(DECODER_CASES):
        d = ThresholdDecoder(cfg, center)
        if d.out_range:
            out['graph_%d' % i] = np.asarray([d.encode(v) for v in np.linspace(0.0, 1.0, 100)[1:-1]], np.float64)
    np.savez_compressed(os.path.join(HERE, 'stats_golden.npz'), **out)
    print('stats_golden.npz', os.path.getsize(os.path.join(HERE, 'stats_golden.npz')), 'fit', mu, std)


if __name__ == '__main__':
    main()
