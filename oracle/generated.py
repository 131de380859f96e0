"""precise-train-generated's sample generator (precise/scripts/train_generated.py:118-226) restated in numpy, two ways.

  literal  the reference's loop: load_audio's float32 x / 32767, calc_volume / normalize_volume_to in float32, the wake-word
           pieces as float64 (layer_with), chunk_audio_pieces and chunk_audio as the reference runs them, merge's
           ``0.4 a + 0.6 b`` (float32 + float64), vals_buffer and max_run_length's decision, consuming the draws it is given
           in the order the reference's lazy generators call random().
  exact    pb_generate's arithmetic bit for bit (include/precise_b200.h): exact int64 sums of squares of the whole background
           and of each whole clip, rms = sqrt(S / n), vol = f rms_bg, g = vol / rms_clip (0 for a silent clip),
           y = 0.4 (f x_bg) + 0.6 (g x_clip) in double with every operation rounded on its own, rint and saturation to int16.

chunk_audio_pieces' ``left_over = piece[-(len(piece) % chunk):]`` runs on layer_with's (2, n) array, so len(piece) is 2 and
left_over is the whole previous piece: each ``combined`` is the previous piece followed by the current one, and chunk_audio
(``range(chunk, len, chunk)``) cuts it into its complete chunks short of the last sample.  An empty previous piece (an empty
clip) is dropped, as ``left_over.size == 0`` drops it.
"""
import math

import numpy as np

I16 = float(np.iinfo(np.int16).max)


# ---- literal ------------------------------------------------------------------------------------------------------------------

def _load(x):
    return np.asarray(x, np.int16).astype(np.float32) / I16


def _rms(a):
    return math.sqrt(np.mean(np.square(a)))


def _to_volume(a, v):
    return v * a / _rms(a)


def _chunks(a, chunk):
    """chunk_audio: [i - chunk, i) for i in range(chunk, len, chunk), along the last axis."""
    n = a.shape[-1]
    return [a[..., i - chunk:i] for i in range(chunk, n, chunk)]


def max_run(x, val):
    """The longest run of ``val`` in x (max_run_length)."""
    best = run = 0
    for v in x:
        run = run + 1 if v == val else 0
        best = max(best, run)
    return best


class Literal:
    """The reference's state across files: the clip cycles, vals_buffer and the draw stream.  ``draws`` is the sequence of
    random() values, consumed in the reference's order, or a function draw(kind, k) -> float with kind 'volume' (k = 0),
    'piece' (k = the file's piece number) or 'save' (k = the file's chunk number)."""

    def __init__(self, wake, other, draws, chunk, sample_rate, buffer_samples, save_prob=0.0):
        self.wake, self.other = [np.asarray(c, np.int16) for c in wake], [np.asarray(c, np.int16) for c in other]
        self.fn = draws if callable(draws) else None
        self.draws, self.k = ([] if callable(draws) else [float(u) for u in draws]), 0   # Python floats, as random()'s
        self.chunk, self.rate, self.save_prob = int(chunk), int(sample_rate), float(save_prob)
        self.vals = np.zeros(int(buffer_samples), np.float64)
        self.next_wake = self.next_other = 0

    def draw(self, kind, k):
        if self.fn is not None:
            return float(self.fn(kind, k))
        u = self.draws[self.k]
        self.k += 1
        return u

    def _pieces(self, volume):
        k = 0
        while True:
            wake = self.draw('piece', k) > 0.5
            if wake:
                clip, self.next_wake = self.wake[self.next_wake], (self.next_wake + 1) % len(self.wake)
            else:
                clip, self.next_other = self.other[self.next_other], (self.next_other + 1) % len(self.other)
            piece = np.empty((2, clip.shape[0]), np.float64)
            piece[0] = _to_volume(_load(clip), volume)
            piece[1] = 1.0 if wake else 0.0
            yield piece
            yield np.zeros((2, int(self.rate * (0.5 + 2.0 * self.draw('piece', k + 1)))), np.float64)
            k += 2

    def _stream(self, volume):
        prev = None
        for piece in self._pieces(volume):
            both = piece if prev is None or prev.size == 0 else np.concatenate([prev, piece], axis=1)
            for c in _chunks(both, self.chunk):
                yield c
            prev = piece

    def file(self, bg):
        """One background file: (merged chunks, float64 [n, chunk]; decisions, int64 [n]: 1, 0 or -1 for skipped).  The
        wake-word stream's chunks (audio and label rows) are left in self.ww, the background's volume in self.volume."""
        audio = _load(bg)
        volume = _rms(audio)
        volume *= 0.4 + 0.5 * self.draw('volume', 0)
        self.volume = volume
        audio = _to_volume(audio, volume)
        merged, decisions, self.ww = [], [], []
        for i, (a, b) in enumerate(zip(_chunks(audio, self.chunk), self._stream(volume))):
            self.ww.append(b)
            merged.append((1.0 - 0.6) * a + 0.6 * b[0])
            self.vals = np.concatenate((self.vals[b.shape[1]:], b[1]))
            frac = max_run(self.vals, 1) / len(self.vals)
            if self.vals[-1] == 0 and frac > 0.8:
                d = 1
            elif frac < 0.5:
                d = 0
            else:
                d = -1
            if d >= 0:
                self.draw('save', i)                                  # the save_prob draw of a kept window
            decisions.append(d)
        return (np.asarray(merged).reshape(-1, self.chunk), np.asarray(decisions, np.int64))


# ---- exact --------------------------------------------------------------------------------------------------------------------

def _sumsq(x):
    return int(np.sum(np.asarray(x, np.int16).astype(np.int64) ** 2))


def _rms_exact(x):
    s = _sumsq(x)
    return math.sqrt(float(s) / float(len(x))) if s > 0 else 0.0


def exact_item(bg, clips, f, length, segments):
    """pb_generate's stream of one item: the first ``length`` samples of background ``bg`` at gain f, overlaid with
    ``segments`` [(clip or -1, first sample, samples)] back to back from sample 0 (they cover at least ``length``)."""
    bg = np.asarray(bg, np.int16)
    f = float(f)
    vol = f * _rms_exact(bg)
    lay = np.zeros(length, np.float64)
    gain = np.zeros(length, np.float64)
    pos = 0
    for c, a, n in segments:
        if pos >= length:
            break
        n = min(int(n), length - pos)
        if c >= 0:
            x = np.asarray(clips[c], np.int16)
            r = _rms_exact(x)
            lay[pos:pos + n] = x[a:a + n]
            gain[pos:pos + n] = vol / r if r > 0 else 0.0
        pos += n
    y = 0.4 * (f * bg[:length].astype(np.float64)) + 0.6 * (gain * lay)
    return np.clip(np.rint(y), -32768, 32767).astype(np.int16)


def exact(backgrounds, clips, items, segments):
    """Every item's stream: items [(background, f, length, first segment, end segment)] over ``segments``."""
    return [exact_item(backgrounds[b], clips, f, int(L), segments[s0:s1]) for b, f, L, s0, s1 in items]
