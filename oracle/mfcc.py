"""Oracle restatement of the MFCC featuriser.  TEST INFRASTRUCTURE ONLY.  ** PARITY UNPINNED **

The arithmetic lives in a third-party dependency that is absent from the reference tree:
``sonopy==0.1.2`` (reference ``requirements.txt:35``; call sites
``precise/vectorization.py:24`` and ``:32-39``).  This file restates sonopy's published
``mfcc_spec`` / ``mel_spec`` / ``power_spec`` / ``filterbanks`` algorithm as the reference
invokes it::

    mfcc_spec(x, pr.sample_rate, (pr.window_samples, pr.hop_samples),
              num_filt=pr.n_filt, fft_size=pr.n_fft, num_coeffs=pr.n_mfcc)

All arithmetic is float64, as in the reference (``Listener.window_audio`` starts as a
float64 array, ``precise/network_runner.py:102,137``).

Semantics restated (each is exercised by a known-answer test in tests/test_oracle_kat.py):
  1. frames: rectangular, ``a[i-W:i] for i in range(W, len(a)+1, hop)`` -- no padding, no
     window function, no pre-emphasis.
  2. ``np.fft.rfft(frames, n=n_fft)``: a frame longer than n_fft is CROPPED to its first
     n_fft samples (numpy semantics), a shorter one is zero padded.
  3. power = (re^2 + im^2) / n_fft.
  4. filterbank: mel(f) = 1127 ln(1 + f/700); grid = linspace(mel(0), mel(sample_rate),
     n_filt + 2) (up to sample_rate, not Nyquist); bin = int(hz * n_bins / sample_rate);
     duplicate grid points are pushed forward; triangle i rises linspace(0,1,mid-left,
     endpoint=False) on [left,mid) and falls linspace(1,0,right-mid,endpoint=False) on
     [mid,right).
  5. mels = log(clip(power @ F.T, eps_f64, None)).
  6. mfcc = DCT-II (norm='ortho') of mels along the filter axis, first n_mfcc columns.
  7. mfcc[:, 0] = log(clip(sum_bins power, eps_f64, None)).
  8. no complete frame -> empty (0, min(n_filt, n_mfcc)) result.
"""
import numpy as np

EPS64 = float(np.finfo(np.float64).eps)


def frame_starts(n_samples: int, window: int, hop: int) -> np.ndarray:
    """Start offsets of every complete frame (semantic 1)."""
    if n_samples < window:
        return np.zeros(0, dtype=np.int64)
    return np.arange(0, n_samples - window + 1, hop, dtype=np.int64)


def power_frames(audio: np.ndarray, window: int, hop: int, n_fft: int) -> np.ndarray:
    """[n_frames, n_fft//2+1] float64 power spectrum (semantics 1-3)."""
    audio = np.asarray(audio, dtype=np.float64)
    starts = frame_starts(len(audio), window, hop)
    n_bins = n_fft // 2 + 1
    if len(starts) == 0:
        return np.zeros((0, n_bins))
    used = min(window, n_fft)          # crop (window > n_fft) or zero-pad (window < n_fft)
    idx = starts[:, None] + np.arange(used)[None, :]
    seg = np.zeros((len(starts), n_fft))
    seg[:, :used] = audio[idx]
    spec = np.fft.rfft(seg, axis=1)
    return (spec.real ** 2 + spec.imag ** 2) / n_fft


def mel_grid(sample_rate: int, n_filt: int, n_bins: int) -> np.ndarray:
    """n_filt+2 FFT-bin indices of the triangle corners (semantic 4), after de-duplication."""
    top = 1127.0 * np.log(1.0 + sample_rate / 700.0)
    mels = np.linspace(0.0, top, n_filt + 2)
    hz = 700.0 * (np.exp(mels / 1127.0) - 1.0)
    raw = (hz * n_bins / sample_rate).astype(int)
    grid = []
    shift = 0
    prev = int(raw[0]) - 1
    for g in raw:
        g = int(g)
        shift = max(0, shift + prev + 1 - g)
        grid.append(g + shift)
        prev = g
    return np.asarray(grid, dtype=np.int64)


def filterbank(sample_rate: int, n_filt: int, n_bins: int) -> np.ndarray:
    """[n_filt, n_bins] triangular mel filter matrix (semantic 4)."""
    grid = mel_grid(sample_rate, n_filt, n_bins)
    bank = np.zeros((n_filt, n_bins))
    for i in range(n_filt):
        lo, mid, hi = int(grid[i]), int(grid[i + 1]), int(grid[i + 2])
        bank[i, lo:mid] = np.linspace(0.0, 1.0, mid - lo, endpoint=False)
        bank[i, mid:hi] = np.linspace(1.0, 0.0, hi - mid, endpoint=False)
    return bank


def dct2_ortho_matrix(n_in: int, n_out: int) -> np.ndarray:
    """D[k, n] such that y = D @ x equals scipy.fftpack.dct(x, type=2, norm='ortho')[:n_out]."""
    n = np.arange(n_in)[None, :]
    k = np.arange(n_out)[:, None]
    d = np.cos(np.pi * k * (2 * n + 1) / (2.0 * n_in)) * np.sqrt(2.0 / n_in)
    d[0, :] *= np.sqrt(0.5)
    return d


def safe_log(x):
    return np.log(np.clip(x, EPS64, None))


def mel_spec(audio, sample_rate, window, hop, n_fft, n_filt) -> np.ndarray:
    """Vectorizer.mels path (reference precise/vectorization.py:32-35)."""
    p = power_frames(audio, window, hop, n_fft)
    return safe_log(p @ filterbank(sample_rate, n_filt, p.shape[1]).T)


def mfcc_spec(audio, sample_rate, window, hop, n_fft, n_filt, n_mfcc) -> np.ndarray:
    """Vectorizer.mfccs path (reference precise/vectorization.py:36-39), semantics 1-8."""
    p = power_frames(audio, window, hop, n_fft)
    n_out = min(n_filt, n_mfcc)
    if p.shape[0] == 0:
        return np.empty((0, n_out))
    mels = safe_log(p @ filterbank(sample_rate, n_filt, p.shape[1]).T)
    out = mels @ dct2_ortho_matrix(n_filt, n_out).T
    out[:, 0] = safe_log(p.sum(axis=1))
    return out


def speechpy_grid(sample_rate: int, n_filt: int, n_bins: int) -> np.ndarray:
    """Corner bins of speechpy.feature.filterbanks as speechpy.feature.mfe calls it: mel points between 0 and sample_rate / 2,
    floor((coefficients + 1) * hz / sample_rate) with coefficients = n_bins (the power spectrum's width)."""
    mels = np.linspace(0.0, 1127.0 * np.log(1.0 + 0.5 * sample_rate / 700.0), n_filt + 2)
    hz = 700.0 * (np.exp(mels / 1127.0) - 1.0)
    return np.floor((n_bins + 1) * hz / sample_rate).astype(np.int64)


def speechpy_mfcc(audio, sample_rate, window, hop, n_fft, n_filt, n_mfcc) -> np.ndarray:
    """Vectorizer.speechpy_mfccs (reference precise/vectorization.py:40-42 -> speechpy.feature.mfcc(x, sample_rate, window_t, hop_t,
    n_mfcc, n_filt, n_fft)).  ** PARITY UNPINNED **: speechpy-fast (setup.py:86) is absent from the reference tree and from this
    image; this restates its published algorithm: stack_frames without zero padding yields floor((len - window) / hop) frames (the
    last complete frame is dropped), rectangular frames, power = |rfft(frame, n_fft)|^2 / n_fft (a longer frame is cropped),
    triangular filters on speechpy_grid (triangle(): rising on (left, middle), falling on [middle, right)), zeros replaced by eps
    before the log, DCT-II (norm='ortho') truncated to n_mfcc, coefficient 0 replaced by the log of the frame energy."""
    audio = np.asarray(audio, dtype=np.float64)
    n_frames = int(np.floor((len(audio) - window) / hop)) if len(audio) >= window else 0
    n_out = min(n_filt, n_mfcc)
    if n_frames <= 0:
        return np.empty((0, n_out))
    p = power_frames(audio[:(n_frames - 1) * hop + window], window, hop, n_fft)
    assert p.shape[0] == n_frames
    grid = speechpy_grid(sample_rate, n_filt, p.shape[1])
    bank = np.zeros((n_filt, p.shape[1]))
    for i in range(n_filt):
        lo, mid, hi = int(grid[i]), int(grid[i + 1]), int(grid[i + 2])
        for k in range(lo + 1, mid):
            bank[i, k] = (k - lo) / (mid - lo)
        for k in range(mid, hi):
            bank[i, k] = (hi - k) / (hi - mid)
    feat = p @ bank.T
    feat[feat == 0] = EPS64
    energy = p.sum(axis=1)
    energy[energy == 0] = EPS64
    out = np.log(feat) @ dct2_ortho_matrix(n_filt, n_out).T
    out[:, 0] = np.log(energy)
    return out


def vectorize_raw(audio, pr) -> np.ndarray:
    """reference precise/vectorization.py:46-50 for Vectorizer.mfccs / Vectorizer.mels / Vectorizer.speechpy_mfccs."""
    if len(audio) == 0:
        raise ValueError('Cannot vectorize empty audio!')   # InvalidAudio is a ValueError (util.py:25)
    if pr.vectorizer == 2:
        return mfcc_spec(audio, pr.sample_rate, pr.window_samples, pr.hop_samples,
                         pr.n_fft, pr.n_filt, pr.n_mfcc)
    if pr.vectorizer == 1:
        return mel_spec(audio, pr.sample_rate, pr.window_samples, pr.hop_samples,
                        pr.n_fft, pr.n_filt)
    if pr.vectorizer == 3:
        return speechpy_mfcc(audio, pr.sample_rate, pr.window_samples, pr.hop_samples, pr.n_fft, pr.n_filt, pr.n_mfcc)
    raise ValueError('unknown vectorizer %r' % (pr.vectorizer,))


def add_deltas(features: np.ndarray) -> np.ndarray:
    """reference precise/vectorization.py:53-59."""
    deltas = np.zeros_like(features)
    deltas[1:] = features[1:] - features[:-1]
    return np.concatenate([features, deltas], -1)


def vectorize(audio, pr) -> np.ndarray:
    """Fixed-length featuriser, reference precise/vectorization.py:62-84."""
    if len(audio) > pr.max_samples:
        audio = audio[-pr.max_samples:]
    feats = vectorize_raw(audio, pr)
    if len(feats) < pr.n_features:
        feats = np.concatenate([np.zeros((pr.n_features - len(feats), feats.shape[1])), feats])
    if len(feats) > pr.n_features:
        feats = feats[-pr.n_features:]
    return feats
