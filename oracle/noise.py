"""precise-add-noise's mix (precise/scripts/add_noise.py:56-90, NoiseData) restated in numpy, two ways.

  exact    pb_add_noise's arithmetic bit for bit: the cyclic noise stream, int64 sums of squares over the raw int16 samples,
           g = r sqrt(Sa) / sqrt(Sn) (0 for a silent span), y = (1 - r) x + g n in double with every operation rounded,
           trunc and saturation to int16.
  literal  the reference's dtypes and operation order: load_audio's float32 x / 32767, the noise as float64 (np.concatenate
           onto np.empty(0)), Python's sequential ``sum`` of ``audio ** 2`` (float32 for the clip, float64 for the noise),
           ``r * (audio_volume * noise / noise_volume) + (1 - r) * audio`` and save_audio's ``(out * 32767).astype(int16)``.

Item i is clip items[i] with ratio ratios[i]; its noise span starts at (pos + the lengths of items 0 .. i-1) mod N, N the
corpus's length, and wraps as often as it needs (get_fresh_noise's read, empty noise files contributing nothing).
"""
import math

import numpy as np


def corpus(noise_clips):
    """The noise files as one int16 stream, in the order given (empty files contribute nothing)."""
    parts = [np.asarray(c, np.int16) for c in noise_clips]
    return np.concatenate(parts + [np.zeros(0, np.int16)])


def span(noise, pos, n):
    """n samples of the cyclic stream from position pos."""
    return noise[(int(pos) + np.arange(n, dtype=np.int64)) % noise.shape[0]]


def positions(lengths, noise_len, pos=0):
    """Each item's noise position and the position after the last item."""
    out = []
    for L in lengths:
        out.append(int(pos))
        pos = (int(pos) + int(L)) % int(noise_len)
    return np.asarray(out, np.int64), int(pos)


def exact_one(x, n, r):
    x = np.asarray(x, np.int16)
    sa = int(np.sum(x.astype(np.int64) ** 2))
    sn = int(np.sum(np.asarray(n, np.int64) ** 2))
    r = float(r)
    g = r * math.sqrt(float(sa)) / math.sqrt(float(sn)) if sn > 0 else 0.0
    y = (1.0 - r) * x.astype(np.float64) + g * np.asarray(n, np.float64)
    return np.clip(np.trunc(y), -32768, 32767).astype(np.int16)


def literal_one(x, n, r):
    r = float(r)                 # random()'s Python float: (1 - r) * audio stays float32, as in the reference
    a = np.asarray(x, np.int16).astype(np.float32) / float(np.iinfo(np.int16).max)
    nd = (np.asarray(n, np.int16).astype(np.float32) / float(np.iinfo(np.int16).max)).astype(np.float64)
    audio_volume = math.sqrt(sum(a ** 2))
    noise_volume = math.sqrt(sum(nd ** 2))
    adjusted = audio_volume * nd / noise_volume
    out = r * adjusted + (1.0 - r) * a
    return (out * np.iinfo(np.int16).max).astype(np.int16)


def volume_ratios(x, n):
    """(exact sqrt(Sa) / sqrt(Sn), literal audio_volume / noise_volume): the noise gain per unit ratio in each form."""
    x = np.asarray(x, np.int16)
    sa = int(np.sum(x.astype(np.int64) ** 2))
    sn = int(np.sum(np.asarray(n, np.int64) ** 2))
    a = x.astype(np.float32) / float(np.iinfo(np.int16).max)
    nd = (np.asarray(n, np.int16).astype(np.float32) / float(np.iinfo(np.int16).max)).astype(np.float64)
    return math.sqrt(float(sa)) / math.sqrt(float(sn)), math.sqrt(sum(a ** 2)) / math.sqrt(sum(nd ** 2))


def _mix(one, clips, noise, items, ratios, pos):
    noise = np.asarray(noise, np.int16)
    if noise.shape[0] == 0:
        raise ValueError('the noise corpus is empty')
    items = [int(i) for i in items]
    starts, end = positions([clips[i].shape[0] for i in items], noise.shape[0], pos)
    return [one(clips[i], span(noise, p, clips[i].shape[0]), r) for i, p, r in zip(items, starts, ratios)], end


def exact(clips, noise, items, ratios, pos=0):
    """pb_add_noise's mixed clips (a list of int16 arrays) and the noise position after them."""
    return _mix(exact_one, clips, noise, items, ratios, pos)


def literal(clips, noise, items, ratios, pos=0):
    """The reference's mixed clips (its dtypes and operation order) and the noise position after them."""
    return _mix(literal_one, clips, noise, items, ratios, pos)
