"""Statistics over labelled clips, restated in numpy: what pb_score_dataset accumulates on the device from the network
outputs, and the expressions of the reference's tools they stand for.

  dataset_stats   the integer statistics (counts per label, the histogram at and between the thresholds, the fixed-point
                  fit sums) of one model's float32 outputs
  calc_threshold  precise/scripts/calc_threshold.py:66-76 in float64
"""
from math import sqrt

import numpy as np


def dataset_stats(outputs, targets, thresholds):
    """outputs float32 [n], targets [n] (non-zero = wake word), thresholds ascending -> (count [2], hist [2, 2 t + 1],
    fit [2, 3]) int64.  Bin 2j + 1 counts outputs == t_j, bin 2j those strictly between t_(j-1) and t_j; NaN goes to bin 0.
    fit: over outputs other than 0 and 1 with a finite v = -log(1 / x - 1) (1 / x - 1 in float32, the log in float64), their
    number, sum(rint(v 2^32)) and sum(rint(v^2 2^24))."""
    x = np.asarray(outputs, np.float32)
    label = np.asarray(targets) != 0
    t = np.asarray(thresholds, np.float32)
    assert np.all(np.diff(t) > 0)
    below = np.searchsorted(t, x, side='left')                # #(t_j < x); NaN sorts last
    below[np.isnan(x)] = 0
    equal = (below < len(t)) & (t[np.minimum(below, len(t) - 1)] == x)
    bins = 2 * below + equal
    count = np.zeros(2, np.int64)
    hist = np.zeros((2, 2 * len(t) + 1), np.int64)
    fit = np.zeros((2, 3), np.int64)
    with np.errstate(all='ignore'):
        v = -np.log((np.float32(1) / x - np.float32(1)).astype(np.float64))
    use = (x != 0) & (x != 1) & np.isfinite(v)
    for l in (0, 1):
        m = label == l
        count[l] = m.sum()
        hist[l] = np.bincount(bins[m], minlength=hist.shape[1])
        vv = v[m & use]
        fit[l] = (vv.size, np.rint(vv * 2.0 ** 32).astype(np.int64).sum(), np.rint(vv * vv * 2.0 ** 24).astype(np.int64).sum())
    return count, hist, fit


def calc_threshold(outputs, targets, smoothing=1.2):
    """(mu, std) as calc_threshold.py:66-76 computes them, in float64; None without data."""
    x = np.asarray(outputs, np.float64)
    tg = np.asarray(targets, np.float64)
    keep = (x != 0) & (x != 1)
    if keep.sum() == 0:
        return None
    inv = -np.log(1 / x[keep] - 1)
    pos = np.extract(tg[keep] > 0.5, inv)
    mu = pos.mean().item()
    return mu, sqrt(np.mean((pos - mu) ** 2)) * smoothing
