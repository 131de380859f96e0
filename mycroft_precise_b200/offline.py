"""Batch / offline callers of the hot path (SURVEY.md 8f rows N2, N3), composed from the same kernels.

  vectorize_raw   ~ precise/vectorization.py:46-50   (whole buffer -> MFCC frames)
  vectorize       ~ precise/vectorization.py:62-84   (crop to the last max_samples, left-zero-pad / crop to n_features rows)
  vectorize_delta ~ precise/vectorization.py:87-89
  evaluate        ~ precise/scripts/simulate.py:92-104 and annoyance_estimator.py:115-130
                    (whole-file MFCC, 29-row windows every chunk_size // hop_samples frames, Runner.predict)

The gather of overlapping windows is a strided view on the device tensor (torch, plumbing); MFCC and
the network run in the CUDA library.

Recorded corpora (many recordings per device call, no window materialised: pb_score_corpus):
  score_corpus      every bank model over a list of recordings, listener or simulate schedule
  score_corpus_pool chosen pool models over a list of recordings (pb_score_corpus_pool)
  score_corpus_pairs chosen (pool model, recording) pairs (pb_score_corpus_pairs)
  Metric, simulate  ~ precise/scripts/simulate.py:45-80, :106-129 (SimulateScript.run's per-file metrics and total)
  simulate_pool     simulate for many pool models in one device call per batch of recordings
  simulate_pairs    simulate for each pool model over its own recordings
  false_activations ~ precise/scripts/train_incremental.py:113-137 (train_on_audio's selection of clips, fixed weights)
  false_activations_pool  the same selection for pool models, the chunks above the threshold found on the device

Labelled clips (one network input per clip, vectorize's; statistics per pool model on the device: pb_score_dataset):
  DatasetStats      ~ precise/stats.py (Stats' counts, rates and format strings, from the device's histograms)
  test_pool         ~ precise/scripts/test.py, eval.py for many pool models in one device call per batch of clips
  graph_thresholds, roc ~ precise/scripts/graph.py:147-152 (the thresholds and the curve precise-graph plots)
  calc_threshold    ~ precise/scripts/calc_threshold.py:66-83 (a model's threshold_config from its positive clips)

Training (up to 128 GRU units, many per call: pb_vectorize_clips, pb_train / pb_train_loss up to 24 units, pb_train_wide /
pb_train_wide_loss beyond):
  vectorize_clips   vectorize(clip) of every clip, on the device
  TrainState, train ~ precise/model.py:57-91, scripts/train.py:159-166 (Keras fit: loss, dropout, RMSprop; val_loss)
  test_rows         test_pool for the networks of a TrainState (up to 128 units), scored from their weight rows
                    (pb_score_rows) over vectorize_clips' inputs

Noise augmentation (pb_add_noise):
  NoiseSource       ~ precise/scripts/add_noise.py:56-80 (NoiseData: the noise files as one cyclic stream and its position)
  add_noise         ~ add_noise.py:82-87 (noised_audio of each clip, on the device)
  vectorize_noisy   vectorize of each noisy clip, without the clips leaving the device
  Augment           fresh noisy copies of every training clip in every epoch of train

Generated training audio (pb_generate, pb_train):
  Generator         ~ precise/scripts/train_generated.py:118-213 (wake words overlaid on backgrounds, windows labelled by
                    vals_buffer's rule), keyed randomness, planned on the host and generated on the device
  train_generated   ~ train_generated.py:215-226 (fit_generator over the generated windows, many networks at once)
"""
from dataclasses import dataclass

import numpy as np

from .core import PB_TRAIN_STRIDE, PB_TRAIN_WIDE_STRIDE, PreciseB200, threshold_encode
from .model_io import GruModel


def _as_device_audio(core: PreciseB200, audio):
    torch = core.torch
    if isinstance(audio, np.ndarray):
        if audio.dtype == np.int16:
            return torch.from_numpy(np.ascontiguousarray(audio)).to(core.device)
        return torch.from_numpy(np.ascontiguousarray(audio, dtype=np.float32)).to(core.device)
    return audio


def vectorize_raw(core: PreciseB200, audio):
    """audio: 1-D (or [S, L]) int16 / float array or CUDA tensor -> [n_frames, F] (or [S, n_frames, F]) CUDA tensor."""
    a = _as_device_audio(core, audio)
    if a.numel() == 0:
        raise ValueError('Cannot vectorize empty audio!')
    one = a.dim() == 1
    out = core.mfcc(a[None] if one else a)
    return out[0] if one else out


def add_deltas(features):
    """[..., T, F] -> [..., T, 2F]; delta[0] = 0 (precise/vectorization.py:53-59)."""
    import torch
    deltas = torch.zeros_like(features)
    deltas[..., 1:, :] = features[..., 1:, :] - features[..., :-1, :]
    return torch.cat([features, deltas], -1)


def vectorize(core: PreciseB200, audio):
    """Fixed-size network input [n_features, F] for one clip (precise/vectorization.py:62-84)."""
    torch = core.torch
    pr = core.params
    a = _as_device_audio(core, audio)
    if a.shape[-1] > pr.max_samples:
        a = a[..., -pr.max_samples:].contiguous()
    feats = vectorize_raw(core, a)
    n = feats.shape[-2]
    if n < pr.n_features:
        pad = torch.zeros(feats.shape[:-2] + (pr.n_features - n, feats.shape[-1]), dtype=feats.dtype, device=feats.device)
        feats = torch.cat([pad, feats], -2)
    if n > pr.n_features:
        feats = feats[..., -pr.n_features:, :]
    return feats


def vectorize_delta(core: PreciseB200, audio):
    return add_deltas(vectorize(core, audio))


def sliding_windows(core: PreciseB200, mfccs, chunk_size_bytes: int):
    """mfccs [n_frames, F] -> [N, n_features, F]: rows i-n_features..i for i in range(n_features, n_frames, hops)
    (simulate.py:96-99; chunk_size is in bytes of int16 audio as everywhere in the reference)."""
    pr = core.params
    hops = chunk_size_bytes // pr.hop_samples
    if hops < 1:
        raise ValueError('chunk_size smaller than one hop')
    T = pr.n_features
    n = mfccs.shape[0]
    ends = range(T, n, hops)
    if len(ends) == 0:
        return mfccs.new_zeros((0, T, mfccs.shape[1]))
    m = mfccs.contiguous()
    F = m.shape[1]
    view = m.as_strided((len(ends), T, F), (hops * F, F, 1))
    return view.contiguous()


def evaluate(core: PreciseB200, audio, chunk_size_bytes: int = 2048):
    """``SimulateScript.evaluate``: network outputs [N] (float32 CUDA tensor) for every window of one recording."""
    mf = vectorize_raw(core, audio)
    win = sliding_windows(core, mf, chunk_size_bytes)
    if core.params.use_delta:
        win = add_deltas(win)
    if win.shape[0] == 0:
        return win.new_zeros((0,))
    return core.predict(win)


# Samples per library call of score_corpus: larger lists are scored in several calls (a single longer recording alone).
CORPUS_CALL_SAMPLES = 1 << 30


def _pack(core: PreciseB200, recs):
    """Recordings -> (1-D int16 device tensor, host int64 offsets [entries + 1], entry index of each recording).  Every
    recording starts at a multiple of 8 samples, so that at the default geometry all its frames take the fast MFCC kernel;
    where the previous one ends elsewhere, an entry of the 1..7 padding samples sits between them (its outputs are dropped)."""
    torch = core.torch
    bounds, entry, pos = [0], [], 0
    for r in recs:
        if pos % 8:
            pos += 8 - pos % 8
            bounds.append(pos)
        entry.append(len(bounds) - 1)
        pos += int(r.shape[0])
        bounds.append(pos)
    offsets = np.asarray(bounds, np.int64)
    pcm = torch.zeros(max(pos, 1), dtype=torch.int16, device=core.device)
    for r, e in zip(recs, entry):
        if r.shape[0]:
            pcm[offsets[e]:offsets[e + 1]].copy_(torch.from_numpy(r) if isinstance(r, np.ndarray) else r)
    return pcm, offsets, np.asarray(entry, np.int64)


def _check_recording(core: PreciseB200, r):
    torch = core.torch
    if isinstance(r, np.ndarray):
        ok = r.dtype == np.int16 and r.ndim == 1
    else:
        ok = isinstance(r, torch.Tensor) and r.dtype == torch.int16 and r.dim() == 1 and r.device == core.device
    if not ok:
        raise ValueError('recordings must be 1-D int16 numpy arrays or CUDA tensors on %s' % core.device)
    return r if isinstance(r, np.ndarray) else r.contiguous()


def _call_groups(recs):
    """Consecutive runs of ``recs`` of at most CORPUS_CALL_SAMPLES samples each (a single longer recording alone)."""
    groups, cur, size = [], [], 0
    for r in recs:
        L = int(r.shape[0])
        if cur and size + L + 8 > CORPUS_CALL_SAMPLES:
            groups.append(cur)
            cur, size = [], 0
        cur.append(r)
        size += L + 8
    groups.append(cur)
    return groups


def _score_groups(core: PreciseB200, recordings, schedule, chunk, call):
    """Packs ``recordings`` into library calls of at most CORPUS_CALL_SAMPLES samples, runs call(pcm, offsets) on each and
    joins the results along the recording axis (window columns for raw / conf / fired, recording columns for the rest).
    Output names score_corpus returns; None outputs stay None."""
    torch = core.torch
    recs = [_check_recording(core, r) for r in recordings]
    groups = _call_groups(recs)
    parts = []
    for g in groups:
        pcm, offsets, entry = _pack(core, g)
        res = call(pcm, offsets)
        if len(entry) < len(offsets) - 1:                     # drop the padding entries
            counts = np.array([core.corpus_windows(int(L), schedule, chunk) for L in np.diff(offsets)], np.int64)
            w0 = np.concatenate([[0], np.cumsum(counts)])
            cols = torch.from_numpy(np.concatenate([np.arange(w0[e], w0[e + 1]) for e in entry] + [np.zeros(0, np.int64)])).to(core.device)
            rows = torch.from_numpy(entry).to(core.device)
            res = {k: None if v is None else v.index_select(1, cols if k in ('raw', 'conf', 'fired') else rows)
                   for k, v in res.items()}
        parts.append(res)
    cat = lambda k: None if parts[0][k] is None else torch.cat([p[k] for p in parts], 1)
    out = {k: cat(k) for k in ('raw', 'conf', 'fired', 'activations', 'above', 'sum')}
    counts = [core.corpus_windows(int(r.shape[0]), schedule, chunk) for r in recs]
    out['window_offsets'] = np.concatenate([[0], np.cumsum(counts, dtype=np.int64)]).astype(np.int64)
    return out


def score_corpus(core: PreciseB200, recordings, schedule='listener', chunk=1024, threshold=0.5, divisor=32768):
    """Every bank model of ``core`` over ``recordings`` (a list of 1-D int16 numpy arrays or CUDA tensors of any lengths).
    Returns dict(raw f32 [M, W], conf f64 [M, W], fired u8 [M, W], window_offsets (host int64 [n + 1]: recording r's windows
    are columns window_offsets[r] .. window_offsets[r + 1] - 1), activations i64 [M, n], and for the simulate schedule
    above i64 [M, n] and sum f64 [M, n], else None).  Schedules: include/precise_b200.h, pb_score_corpus.  divisor: 32768 for
    audio as the stream path reads it (buffer_to_audio), 32767 for audio as load_audio reads wav files."""
    return _score_groups(core, recordings, schedule, chunk,
                         lambda pcm, offsets: core.score_corpus(pcm, offsets, schedule, chunk, threshold, divisor))


def score_corpus_pool(core: PreciseB200, recordings, model_ids, schedule='listener', chunk=1024, threshold=0.5, divisor=32768,
                      per_window=True):
    """score_corpus for pool models ``model_ids`` (int32 [k], repeats allowed): the same dict with k rows in the order of
    model_ids.  per_window=False: raw, conf and fired are None, only the reductions are computed (pb_score_corpus_pool)."""
    ids = np.ascontiguousarray(model_ids, dtype=np.int32)
    return _score_groups(core, recordings, schedule, chunk,
                         lambda pcm, offsets: core.score_corpus_pool(pcm, offsets, ids, schedule, chunk, threshold, divisor,
                                                                     per_window))


def score_corpus_pairs(core: PreciseB200, recordings, model_ids, rec_ids, schedule='listener', chunk=1024, threshold=0.5,
                       divisor=32768, per_window=True, hit_threshold=None, hit_capacity=None):
    """Pool model model_ids[p] over recordings[rec_ids[p]] for each pair p (pb_score_corpus_pairs), recordings packed and
    split into library calls as score_corpus splits them; each call scores the pairs whose recordings it holds.  Returns
    PreciseB200.score_corpus_pairs's dict over all pairs, in pair order: raw / conf / fired [Wp] (None with
    per_window=False), activations (and for simulate above, sum) [n_pairs], pair_offsets, and hits with a hit_threshold."""
    torch = core.torch
    recs = [_check_recording(core, r) for r in recordings]
    model_ids = np.ascontiguousarray(model_ids, dtype=np.int32)
    rec_ids = np.ascontiguousarray(rec_ids, dtype=np.int64)
    n = model_ids.shape[0]
    if rec_ids.shape != (n,):
        raise ValueError('model_ids and rec_ids must be 1-D arrays of one length')
    if n and (rec_ids.min() < 0 or rec_ids.max() >= len(recs)):
        raise ValueError('recording ids must lie in [0, %d)' % len(recs))
    counts = np.asarray([core.corpus_windows(int(r.shape[0]), schedule, chunk) for r in recs], np.int64)
    P = np.concatenate([[0], np.cumsum(counts[rec_ids], dtype=np.int64)]).astype(np.int64)
    Wp = int(P[-1])
    parts, first = [], 0
    for g in _call_groups(recs):
        sel = np.nonzero((rec_ids >= first) & (rec_ids < first + len(g)))[0]
        if sel.size:
            pcm, offsets, entry = _pack(core, g)
            res = core.score_corpus_pairs(pcm, offsets, model_ids[sel], entry[rec_ids[sel] - first].astype(np.int32),
                                          schedule, chunk, threshold, divisor, per_window, hit_threshold, hit_capacity)
            parts.append((sel, res))
        first += len(g)
    if len(parts) == 1 and parts[0][0].size == n:                # one call over every pair, in order
        res = parts[0][1]
        res['pair_offsets'] = P
        return res
    f = lambda size, dt: torch.zeros(size, dtype=dt, device=core.device)
    out = dict(raw=None, conf=None, fired=None, activations=f(n, torch.int64), above=None, sum=None, pair_offsets=P)
    if per_window:
        out.update(raw=f(Wp, torch.float32), conf=f(Wp, torch.float64), fired=f(Wp, torch.uint8))
    if schedule == 'simulate':
        out.update(above=f(n, torch.int64), sum=f(n, torch.float64))
    hits = []
    for sel, res in parts:
        rows = torch.from_numpy(sel).to(core.device)
        for k in ('activations', 'above', 'sum'):
            if out[k] is not None:
                out[k].index_copy_(0, rows, res[k])
        local = res['pair_offsets']
        if per_window:                                           # this call's pair-windows, placed at their pairs' columns
            cols = np.concatenate([np.arange(P[p], P[p + 1]) for p in sel] + [np.zeros(0, np.int64)])
            cols = torch.from_numpy(cols).to(core.device)
            for k in ('raw', 'conf', 'fired'):
                out[k].index_copy_(0, cols, res[k])
        if hit_threshold is not None:
            q = res['hits'].cpu().numpy()
            j = np.searchsorted(local, q, side='right') - 1
            hits.append(P[sel[j]] + (q - local[j]))
    if hit_threshold is not None:
        out['hits'] = torch.from_numpy(np.sort(np.concatenate(hits + [np.zeros(0, np.int64)]))).to(core.device)
    return out


@dataclass
class Metric:
    """precise-simulate's false-activation metric of one recording or of a whole folder (simulate.py:45-80)."""
    chunk_size: int
    seconds: float = 0.0
    activated_chunks: int = 0
    activations: int = 0
    activation_sum: float = 0.0
    sample_rate: int = 16000

    @property
    def days(self) -> float:
        return self.seconds / 86400.0

    @property
    def chunks(self) -> float:
        return self.seconds * self.sample_rate / self.chunk_size

    def add(self, other: 'Metric'):
        self.seconds += other.seconds
        self.activated_chunks += other.activated_chunks
        self.activations += other.activations
        self.activation_sum += other.activation_sum

    def info_string(self, title: str) -> str:
        lines = ['=== %s ===' % title,
                 'Hours: {:.2f}'.format(self.days * 24),
                 'Activations / Day: {:.2f}'.format(self.activations / self.days),
                 'Activated Chunks / Day: {:.2f}'.format(self.activated_chunks / self.days),
                 'Average Activation (*100): {:.2f}'.format(100.0 * self.activation_sum / self.chunks)]
        return '\n'.join(lines)


def simulate(core: PreciseB200, recordings, chunk_size=4096, threshold=0.5):
    """SimulateScript.run's numbers for bank slot 0 over int16 recordings read as load_audio reads them (samples / 32767):
    (one Metric per recording, their total).  An empty recording is skipped, as the reference skips it: its entry is None.
    A recording too short for one window (fewer than n_features + 1 frames) counts its seconds with no windows, where the
    reference's Runner.predict fails on an empty input."""
    res = score_corpus(core, recordings, 'simulate', chunk_size, threshold, divisor=32767)
    return _metrics(core, recordings, chunk_size, res['above'][0].cpu().numpy(), res['activations'][0].cpu().numpy(),
                    res['sum'][0].cpu().numpy())


def _metrics(core: PreciseB200, recordings, chunk_size, above, acts, sums):
    """Per-recording Metrics of one model (None for an empty recording) and their total."""
    sr = core.params.sample_rate
    total = Metric(chunk_size, sample_rate=sr)
    metrics = []
    for i, r in enumerate(recordings):
        L = int(r.shape[0])
        if L == 0:
            metrics.append(None)
            continue
        m = Metric(chunk_size, L / sr, int(above[i]), int(acts[i]), float(sums[i]), sr)
        total.add(m)
        metrics.append(m)
    return metrics, total


def simulate_pool(core: PreciseB200, recordings, model_ids, chunk_size=4096, threshold=0.5):
    """simulate for many pool models on one K1: returns (metrics, totals), metrics[i][r] model_ids[i]'s Metric for recording
    r (None for an empty recording) and totals[i] its total.  Only the per-recording reductions leave the device."""
    res = score_corpus_pool(core, recordings, model_ids, 'simulate', chunk_size, threshold, divisor=32767, per_window=False)
    above = res['above'].cpu().numpy()
    acts = res['activations'].cpu().numpy()
    sums = res['sum'].cpu().numpy()
    metrics, totals = [], []
    for i in range(above.shape[0]):
        m, t = _metrics(core, recordings, chunk_size, above[i], acts[i], sums[i])
        metrics.append(m)
        totals.append(t)
    return metrics, totals


def simulate_pairs(core: PreciseB200, recordings, model_ids, rec_ids, chunk_size=4096, threshold=0.5):
    """simulate for chosen (pool model, recording) pairs, each custom wake word over its own recordings: returns (metrics,
    totals), metrics[p] pair p's Metric (None for an empty recording) and totals {model id: the total over its pairs, in
    pair order}.  Only the per-pair reductions leave the device."""
    res = score_corpus_pairs(core, recordings, model_ids, rec_ids, 'simulate', chunk_size, threshold, divisor=32767,
                             per_window=False)
    above = res['above'].cpu().numpy()
    acts = res['activations'].cpu().numpy()
    sums = res['sum'].cpu().numpy()
    sr = core.params.sample_rate
    metrics, totals = [], {}
    for p, (mid, r) in enumerate(zip(np.asarray(model_ids).tolist(), np.asarray(rec_ids).tolist())):
        t = totals.setdefault(mid, Metric(chunk_size, sample_rate=sr))
        L = int(recordings[r].shape[0])
        if L == 0:
            metrics.append(None)
            continue
        m = Metric(chunk_size, L / sr, int(above[p]), int(acts[p]), float(sums[p]), sr)
        t.add(m)
        metrics.append(m)
    return metrics, totals


def false_activations(core: PreciseB200, recordings, chunk_size=2048, threshold=0.5):
    """train_on_audio's selection (train_incremental.py:113-137) with fixed weights, bank slot 0, recordings read as
    load_audio reads them (samples / 32767).  Each recording is cut as chunk_audio cuts it (util.py:30-32: chunks end at
    range(c, L, c), floor((L - 1) / c) of them) and fed to a fresh listener of chunk c.  Returns a list of (recording index,
    chunk index, clip) for every chunk whose confidence is above ``threshold``; the clip is the float32 audio of the last
    buffer_samples samples up to the end of that chunk, zeros before the recording's start.
    Deliberate differences: the reference's audio_buffer carries the previous file's tail into the next file (glob order),
    here every recording starts from zeros; and it retrains between chunks, which is out of scope here."""
    c = int(chunk_size)
    recs = _chunk_cut(recordings, c)
    res = score_corpus(core, recs, 'listener', c, divisor=32767)
    conf = res['conf'][0].cpu().numpy()
    wo = res['window_offsets']
    bs = core.params.buffer_samples
    out = []
    for i, r in enumerate(recs):
        hits = np.nonzero(conf[wo[i]:wo[i + 1]] > threshold)[0]
        if hits.size == 0:
            continue
        a = r if isinstance(r, np.ndarray) else r.cpu().numpy()
        for k in hits:
            out.append((i, int(k), _clip(a, (int(k) + 1) * c, bs)))
    return out


def _chunk_cut(recordings, c):
    """Each recording cut as chunk_audio cuts it (util.py:30-32): floor((L - 1) / c) chunks of c."""
    return [r[:((int(r.shape[0]) - 1) // c) * c] if int(r.shape[0]) else r for r in recordings]


def _clip(a, end, bs):
    """The float32 audio (load_audio's scale) of the last bs samples of ``a`` up to ``end``, zeros before its start."""
    clip = np.zeros(bs, np.float32)
    seg = a[max(0, end - bs):end].astype(np.float32) / np.float32(32767)
    clip[bs - seg.shape[0]:] = seg
    return clip


def false_activations_pool(core: PreciseB200, recordings, model_ids, rec_ids=None, chunk_size=2048, threshold=0.5):
    """false_activations for pool models: pool model model_ids[p] over recordings[rec_ids[p]] for each pair p (rec_ids None:
    every model over every recording, model-major, pair p = i * len(recordings) + r).  Recordings are cut and clips built as
    false_activations does; the chunks above ``threshold`` are found on the device, and only they leave it.  Returns a list
    of (pair index, recording index, chunk index, clip), in pair order and chunk order within a pair."""
    c = int(chunk_size)
    recs = _chunk_cut(recordings, c)
    model_ids = np.ascontiguousarray(model_ids, dtype=np.int32)
    if rec_ids is None:
        n_rec = len(recs)
        rec_ids = np.tile(np.arange(n_rec, dtype=np.int32), model_ids.shape[0])
        model_ids = np.repeat(model_ids, n_rec)
    rec_ids = np.ascontiguousarray(rec_ids, dtype=np.int32)
    res = score_corpus_pairs(core, recs, model_ids, rec_ids, 'listener', c, divisor=32767, per_window=False,
                             hit_threshold=threshold)
    P = res['pair_offsets']
    q = res['hits'].cpu().numpy()
    pair = np.searchsorted(P, q, side='right') - 1
    bs = core.params.buffer_samples
    host = {}
    out = []
    for p, k in zip(pair.tolist(), (q - P[pair]).tolist()):
        r = int(rec_ids[p])
        if r not in host:
            a = recs[r]
            host[r] = a if isinstance(a, np.ndarray) else a.cpu().numpy()
        out.append((p, r, k, _clip(host[r], (k + 1) * c, bs)))
    return out


COUNTS_STR = """=== Counts ===
False Positives: {false_pos}
True Negatives: {true_neg}
False Negatives: {false_neg}
True Positives: {true_pos}"""

SUMMARY_STR = """
=== Summary ===
{num_correct} out of {total}
{accuracy_ratio:.2%}

{false_pos_ratio:.2%} false positives
{false_neg_ratio:.2%} false negatives
"""


class DatasetStats:
    """One model's statistics over labelled clips, as pb_score_dataset returns them: count [2] (clips per label, 1 = wake
    word), hist [2, 2 n + 1] (the outputs binned at and between the n float32 thresholds) and fit [2, 3] (calc_threshold's
    sums), all int64.  It answers what precise/stats.py's Stats answers from the outputs themselves, at the thresholds the
    call was given: any other threshold raises KeyError.  Two DatasetStats over the same thresholds add."""

    def __init__(self, thresholds, count, hist, fit):
        self.thresholds = np.asarray(thresholds, np.float32)
        self.count = np.asarray(count, np.int64)
        self.hist = np.asarray(hist, np.int64)
        self.fit = np.asarray(fit, np.int64)
        if self.count.shape != (2,) or self.hist.shape != (2, 2 * self.thresholds.shape[0] + 1) or self.fit.shape != (2, 3):
            raise ValueError('count [2], hist [2, 2 n_thr + 1] and fit [2, 3] expected')

    def __add__(self, other):
        if not np.array_equal(self.thresholds, other.thresholds):
            raise ValueError('statistics over different thresholds do not add')
        return DatasetStats(self.thresholds, self.count + other.count, self.hist + other.hist, self.fit + other.fit)

    def __len__(self):
        return int(self.count.sum())

    def _above(self, label, threshold, equal):
        """#(output > threshold) of one label, or with ``equal`` #(output >= threshold); float32 comparisons, as numpy's."""
        t = np.float32(threshold)
        j = int(np.searchsorted(self.thresholds, t))
        if j == self.thresholds.shape[0] or self.thresholds[j] != t:
            raise KeyError('threshold %r is not one of this call\'s' % (threshold,))
        return int(self.hist[label, 2 * j + (1 if equal else 2):].sum())

    def true_pos(self, threshold=0.5):
        return self._above(1, threshold, False)

    def false_pos(self, threshold=0.5):
        return self._above(0, threshold, False)

    def true_neg(self, threshold=0.5):
        return int(self.count[0]) - self.false_pos(threshold)

    def false_neg(self, threshold=0.5):
        return int(self.count[1]) - self.true_pos(threshold)

    def false_positives(self, threshold=0.5):
        return self.false_pos(threshold) / max(1, int(self.count[0]))

    def false_negatives(self, threshold=0.5):
        return self.false_neg(threshold) / max(1, int(self.count[1]))

    def num_correct(self, threshold=0.5):
        """Stats.num_correct (stats.py:54-56) compares with >=, where the counts above compare with >."""
        return self._above(1, threshold, True) + int(self.count[0]) - self._above(0, threshold, True)

    def num_incorrect(self, threshold=0.5):
        return len(self) - self.num_correct(threshold)

    def accuracy(self, threshold=0.5):
        return self.num_correct(threshold) / max(1, len(self))

    def counts_str(self, threshold=0.5):
        return COUNTS_STR.format(false_pos=self.false_pos(threshold), true_neg=self.true_neg(threshold),
                                 false_neg=self.false_neg(threshold), true_pos=self.true_pos(threshold))

    def summary_str(self, threshold=0.5):
        return SUMMARY_STR.format(num_correct=self.num_correct(threshold), total=len(self),
                                  accuracy_ratio=self.accuracy(threshold), false_pos_ratio=self.false_positives(threshold),
                                  false_neg_ratio=self.false_negatives(threshold))


def _pack_clips(core: PreciseB200, clips):
    """Clips -> (1-D int16 device tensor, host int64 offsets [n + 1], clip index of each entry), each clip cropped to the
    last max_samples samples the network sees and packed back to back: pb_score_dataset's cross product scores every entry,
    so there are no padding entries.  Clips whose length is a multiple of 8 samples go first, so that all of them start
    aligned and take the fast MFCC kernel at the default geometry."""
    torch = core.torch
    ms = core.params.max_samples
    clips = [c[-ms:] if int(c.shape[0]) > ms else c for c in clips]
    order = sorted(range(len(clips)), key=lambda i: int(clips[i].shape[0]) % 8 != 0)
    offsets = np.concatenate([[0], np.cumsum([int(clips[i].shape[0]) for i in order], dtype=np.int64)]).astype(np.int64)
    pcm = torch.zeros(max(int(offsets[-1]), 1), dtype=torch.int16, device=core.device)
    for e, i in enumerate(order):
        c = clips[i]
        pcm[offsets[e]:offsets[e + 1]].copy_(torch.from_numpy(np.ascontiguousarray(c)) if isinstance(c, np.ndarray) else c)
    return pcm, offsets, np.asarray(order, np.int64)


def test_pool(core: PreciseB200, clips, targets, model_ids, rows=None, recs=None, thresholds=(0.5,), misses=False,
              miss_threshold=0.5):
    """precise-test's statistics for pool models ``model_ids`` (int32 [k]) over labelled ``clips`` (1-D int16 numpy arrays or
    CUDA tensors read as load_audio reads them, none empty; targets[c] non-zero = wake word).  rows / recs None: every model
    over every clip.  Otherwise entry p is model_ids[rows[p]] over clips[recs[p]]: each word over its owner's clips.  Clips
    are split into library calls as score_corpus splits recordings, and the calls' statistics are added.  Returns a list of
    k DatasetStats; with misses=True also a list of k sorted arrays, the clip indices model i misclassifies at
    ``miss_threshold`` ((output > miss_threshold) != label, Stats.calc_filenames' rule).  Only statistics and misclassified
    indices leave the device."""
    clips = [_check_recording(core, c) for c in clips]
    targets = np.ascontiguousarray(np.asarray(targets) != 0, dtype=np.uint8)
    model_ids = np.ascontiguousarray(model_ids, dtype=np.int32)
    if targets.shape != (len(clips),):
        raise ValueError('one target per clip')
    k = model_ids.shape[0]
    if (rows is None) != (recs is None):
        raise ValueError('rows and recs come together')
    if rows is not None:
        rows, recs = np.ascontiguousarray(rows, dtype=np.int32), np.ascontiguousarray(recs, dtype=np.int64)
        if rows.ndim != 1 or rows.shape != recs.shape:
            raise ValueError('rows and recs must be 1-D arrays of one length')
        if rows.size and (recs.min() < 0 or recs.max() >= len(clips) or rows.min() < 0 or rows.max() >= k):
            raise ValueError('rows must lie in [0, %d) and recs in [0, %d)' % (k, len(clips)))
    thr = np.unique(np.asarray(thresholds, np.float32))
    n_thr = thr.shape[0]
    count, hist, fit = np.zeros((k, 2), np.int64), np.zeros((k, 2, 2 * n_thr + 1), np.int64), np.zeros((k, 2, 3), np.int64)
    missed = [[] for _ in range(k)]
    first = 0
    for g in _call_groups(clips):
        pcm, offsets, order = _pack_clips(core, g)
        entry = np.empty(len(g), np.int64)                    # clip (within the group) -> entry of the call
        entry[order] = np.arange(len(g))
        tg = np.ascontiguousarray(targets[first + order])
        kw = dict(thresholds=thr.astype(np.float64), per_entry=False, miss_threshold=miss_threshold if misses else None)
        if rows is None:
            res = core.score_dataset(pcm, offsets, tg, model_ids, **kw)
        else:
            sel = np.nonzero((recs >= first) & (recs < first + len(g)))[0]
            res = core.score_dataset(pcm, offsets, tg, model_ids, rows[sel], entry[recs[sel] - first].astype(np.int32), **kw)
        count += res['count'].cpu().numpy()
        hist += res['hist'].cpu().numpy()
        fit += res['fit'].cpu().numpy()
        if misses:
            q = res['misses'].cpu().numpy()
            if rows is None:
                for i, e in zip((q // len(g)).tolist(), (q % len(g)).tolist()):
                    missed[i].append(first + int(order[e]))
            else:
                for p in sel[q].tolist():
                    missed[int(rows[p])].append(int(recs[p]))
        first += len(g)
    stats = [DatasetStats(thr, count[i], hist[i], fit[i]) for i in range(k)]
    if misses:
        return stats, [np.asarray(sorted(m), np.int64) for m in missed]
    return stats


test_pool.__test__ = False        # not a pytest test, whatever module imports it


def graph_thresholds(params, resolution=100):
    """The network outputs precise-graph evaluates (graph.py:147-148): ThresholdDecoder.encode of
    linspace(0, 1, resolution)[1:-1] under the model's threshold_config and center, sorted and de-duplicated in float32 (the
    precision the outputs are compared in)."""
    enc = threshold_encode(params.threshold_config, params.threshold_center, np.linspace(0.0, 1.0, resolution)[1:-1])
    return np.unique(enc.astype(np.float32))


def roc(stats: DatasetStats):
    """(false-positive rates, false-negative rates) over the statistics' thresholds, ascending: precise-graph's x and y."""
    t = stats.thresholds
    return (np.asarray([stats.false_positives(v) for v in t]), np.asarray([stats.false_negatives(v) for v in t]))


def calc_threshold(stats: DatasetStats, smoothing=1.2):
    """precise-calc-threshold's (mu, std) (calc_threshold.py:66-76) from the wake-word clips' fit sums: the mean of
    v = -log(1 / output - 1) over outputs other than 0 and 1, and sqrt(mean(v^2) - mu^2) * smoothing; the model's
    threshold_config is ((mu, std),).  None when no wake-word clip's output lies strictly between 0 and 1 (the reference
    prints "No data").  The reference computes v and both means in float32; here v is a double (of the float32
    1 / output - 1) summed in fixed point, exact to 2^-32 in mu."""
    n, s1, s2 = (int(v) for v in stats.fit[1])
    if n == 0:
        return None
    mu = s1 / 2.0 ** 32 / n
    var = s2 / 2.0 ** 24 / n - mu * mu
    return mu, float(np.sqrt(max(var, 0.0))) * smoothing


# ---- training ---------------------------------------------------------------------------------------------------------------

def vectorize_clips(core: PreciseB200, clips, divisor=32767):
    """vectorize(clip) of every clip (1-D int16 numpy arrays or CUDA tensors, none empty; divisor 32767: read as load_audio
    reads wav files) -> float32 CUDA tensor [n, n_features, feature_size], bit for bit the input score_dataset scores.  Clips
    are split into library calls as test_pool splits them."""
    clips = [_check_recording(core, c) for c in clips]
    parts = []
    for g in _call_groups(clips):
        pcm, offsets, order = _pack_clips(core, g)
        res = core.vectorize_clips(pcm, offsets, divisor)
        out = core.torch.empty_like(res)
        out[core.torch.from_numpy(order).to(core.device)] = res
        parts.append(out)
    if not parts:
        return core.torch.empty((0, core.n_features, core.feature_size), dtype=core.torch.float32, device=core.device)
    return core.torch.cat(parts) if len(parts) > 1 else parts[0]


class TrainState:
    """Networks being trained on one handle's front end: their weights and RMSprop accumulators as device rows
    [k, stride] (Keras's order: kernel, recurrent, bias, dense_w, dense_b), each row's hidden size, activations and
    seed, and the next epoch's number (the shuffles and dropout masks of a resumed fit continue from it).  ``stride`` is the
    layout: PB_TRAIN_STRIDE (pb_train) when every network has at most 24 units, else PB_TRAIN_WIDE_STRIDE (pb_train_wide, up
    to 128 units); the training calls follow the rows' width."""

    def __init__(self, core: PreciseB200, weights, rms, hidden, activation, recurrent_activation, seeds, epoch=0):
        self.core = core
        self.weights, self.rms = weights, rms
        self.hidden, self.activation, self.recurrent_activation = list(hidden), list(activation), list(recurrent_activation)
        self.seeds = [int(s) for s in seeds]
        self.epoch = int(epoch)
        self.rows = core.train_rows(self.hidden, self.activation, self.recurrent_activation, self.seeds)
        k = len(self.hidden)
        self.stride = PB_TRAIN_WIDE_STRIDE if k and weights.numel() == k * PB_TRAIN_WIDE_STRIDE else PB_TRAIN_STRIDE

    @property
    def wide(self):
        """Whether the rows have pb_train_wide's layout."""
        return self.stride == PB_TRAIN_WIDE_STRIDE

    @staticmethod
    def from_models(core: PreciseB200, models, seeds):
        """One row per GruModel (feature size core.feature_size, hidden <= 128), accumulators at zero; the wide layout when
        any network has more than 24 units."""
        torch = core.torch
        wide = any(m.hidden > 24 for m in models)
        w = np.zeros((len(models), PB_TRAIN_WIDE_STRIDE if wide else PB_TRAIN_STRIDE), np.float32)
        for i, m in enumerate(models):
            if m.feature_size != core.feature_size:
                raise ValueError('model %d has feature size %d, the handle %d' % (i, m.feature_size, core.feature_size))
            flat = np.concatenate([m.kernel.ravel(), m.recurrent.ravel(), m.bias, m.dense_w, [np.float32(m.dense_b)]])
            w[i, :flat.size] = flat
        weights = torch.from_numpy(w).to(core.device)
        return TrainState(core, weights, torch.zeros_like(weights), [m.hidden for m in models], [m.activation for m in models],
                          [m.recurrent_activation for m in models], seeds)

    def models(self):
        """The current weights as GruModels."""
        w = self.weights.cpu().numpy()
        F = self.core.feature_size
        out = []
        for i, H in enumerate(self.hidden):
            a = 0
            parts = []
            for n in (3 * H * F, 3 * H * H, 3 * H, H, 1):
                parts.append(w[i, a:a + n])
                a += n
            out.append(GruModel(parts[0].reshape(F, 3 * H), parts[1].reshape(H, 3 * H), parts[2], parts[3], parts[4],
                                self.activation[i], self.recurrent_activation[i]))
        return out


# Clips per pb_score_rows call of test_rows: the fit's sums hold 2^24 entries of one (row, label).
ROWS_CALL_CLIPS = 1 << 24


def test_rows(core: PreciseB200, state: TrainState, inputs, targets, rows=None, recs=None, thresholds=(0.5,), misses=False,
              miss_threshold=0.5):
    """test_pool for the networks of ``state`` (a TrainState, or TrainState.from_models(core, models, seeds) for models on
    disk; up to 128 units), scored straight from its weight rows (pb_score_rows) over ``inputs`` (vectorize_clips' tensor)
    with labels ``targets`` (non-zero = wake word).  rows / recs None: every network over every input; otherwise entry p is
    network rows[p] over inputs[recs[p]].  Inputs are split into calls of at most ROWS_CALL_CLIPS clips and the calls'
    statistics are added.  Returns a list of k DatasetStats, and with misses=True also a list of k sorted arrays of the
    input indices network i misclassifies at ``miss_threshold``, as test_pool does."""
    targets = np.ascontiguousarray(np.asarray(targets) != 0, dtype=np.uint8)
    n_rec, k = int(inputs.shape[0]), len(state.hidden)
    if targets.shape != (n_rec,):
        raise ValueError('one target per input')
    if (rows is None) != (recs is None):
        raise ValueError('rows and recs come together')
    if rows is not None:
        rows, recs = np.ascontiguousarray(rows, dtype=np.int32), np.ascontiguousarray(recs, dtype=np.int64)
        if rows.ndim != 1 or rows.shape != recs.shape:
            raise ValueError('rows and recs must be 1-D arrays of one length')
        if rows.size and (recs.min() < 0 or recs.max() >= n_rec or rows.min() < 0 or rows.max() >= k):
            raise ValueError('rows must lie in [0, %d) and recs in [0, %d)' % (k, n_rec))
    thr = np.unique(np.asarray(thresholds, np.float32))
    n_thr = thr.shape[0]
    count, hist, fit = np.zeros((k, 2), np.int64), np.zeros((k, 2, 2 * n_thr + 1), np.int64), np.zeros((k, 2, 3), np.int64)
    missed = [[] for _ in range(k)]
    kw = dict(thresholds=thr.astype(np.float64), per_entry=False, miss_threshold=miss_threshold if misses else None)
    for c0 in range(0, n_rec, ROWS_CALL_CLIPS):
        c1 = min(n_rec, c0 + ROWS_CALL_CLIPS)
        if rows is None:
            res = core.score_rows(inputs[c0:c1], targets[c0:c1], state.rows, state.weights, **kw)
        else:
            sel = np.nonzero((recs >= c0) & (recs < c1))[0]
            res = core.score_rows(inputs[c0:c1], targets[c0:c1], state.rows, state.weights, rows[sel],
                                  (recs[sel] - c0).astype(np.int32), **kw)
        count += res['count'].cpu().numpy()
        hist += res['hist'].cpu().numpy()
        fit += res['fit'].cpu().numpy()
        if misses:
            q = res['misses'].cpu().numpy()
            if rows is None:
                for i, r in zip((q // (c1 - c0)).tolist(), (q % (c1 - c0)).tolist()):
                    missed[i].append(c0 + r)
            else:
                for p in sel[q].tolist():
                    missed[int(rows[p])].append(int(recs[p]))
    stats = [DatasetStats(thr, count[i], hist[i], fit[i]) for i in range(k)]
    if misses:
        return stats, [np.asarray(sorted(m), np.int64) for m in missed]
    return stats


test_rows.__test__ = False        # not a pytest test, whatever module imports it


def train(core: PreciseB200, state: TrainState, inputs, targets, rows=None, recs=None, epochs=10, batch_size=5000,
          sensitivity=0.2, dropout=0.2, lr=0.001, validation=None, augment=None):
    """precise-train's fit for every network of ``state`` at once (pb_train): ``epochs`` epochs over ``inputs``
    (vectorize_clips' tensor) with labels ``targets`` (non-zero = wake word), loss_bias = 1 - sensitivity (train.py:86).
    rows / recs None: every network on every input; otherwise entry p is inputs[recs[p]] for network rows[p] (each word
    on its owner's clips plus shared negatives).  state.epoch advances by ``epochs``.  Returns the epoch losses, float64
    [k, epochs]; with validation=(inputs, targets) or (inputs, targets, rows, recs) also val_loss [k, epochs], each
    network's loss over its validation entries without dropout after each epoch (pb_train_loss, Keras's evaluate).
    augment (an Augment): ``inputs`` are then the clips themselves (as vectorize_clips takes them), and each epoch is one
    pb_train call over entries clip-major, clip c's clean input at c (copies + 1) followed by its noisy copies; targets
    and rows / recs pairs expand to each clip's clean and noisy entries.  Validation stays clean."""
    kw = dict(rows_of=rows, recs=recs, batch_size=batch_size, lr=lr, loss_bias=1.0 - sensitivity, dropout=dropout)
    if augment is not None:
        vals = []
        step = lambda: None
        if validation is not None:
            v_in, v_tg = validation[0], validation[1]
            v_rows, v_recs = (validation[2], validation[3]) if len(validation) > 2 else (None, None)
            step = lambda: vals.append(core.train_loss(v_in, v_tg, state.rows, state.weights, v_rows, v_recs,
                                                       loss_bias=1.0 - sensitivity))
        kw.pop('rows_of'), kw.pop('recs')
        loss = _train_augmented(core, state, inputs, targets, rows, recs, epochs, kw, augment, step)
        if validation is None:
            return loss
        return loss, core.torch.stack(vals, 1).cpu().numpy() if vals else np.zeros((len(state.hidden), 0))
    if validation is None:
        loss = core.train(inputs, targets, state.rows, state.weights, state.rms, epochs=epochs, epoch0=state.epoch, **kw)
        state.epoch += epochs
        return loss.cpu().numpy()
    v_in, v_tg = validation[0], validation[1]
    v_rows, v_recs = (validation[2], validation[3]) if len(validation) > 2 else (None, None)
    losses, vals = [], []
    for _ in range(epochs):
        losses.append(core.train(inputs, targets, state.rows, state.weights, state.rms, epochs=1, epoch0=state.epoch, **kw))
        state.epoch += 1
        vals.append(core.train_loss(v_in, v_tg, state.rows, state.weights, v_rows, v_recs, loss_bias=1.0 - sensitivity))
    k = len(state.hidden)
    loss = core.torch.cat(losses, 1).cpu().numpy() if losses else np.zeros((k, 0))
    val = core.torch.stack(vals, 1).cpu().numpy() if vals else np.zeros((k, 0))
    return loss, val


# ---- noise augmentation -----------------------------------------------------------------------------------------------------

class NoiseSource:
    """A noise corpus packed on the device as one int16 stream (the clips in the order given; empty ones contribute
    nothing), and ``pos``, the position NoiseData.get_fresh_noise reads on from (add_noise.py:56-80).  add_noise and
    vectorize_noisy advance it by the lengths of the clips they mix, modulo the corpus's length."""

    def __init__(self, core: PreciseB200, noise_clips, pos=0):
        torch = core.torch
        clips = [_check_recording(core, c) for c in noise_clips]
        parts = [torch.from_numpy(np.ascontiguousarray(c)) if isinstance(c, np.ndarray) else c for c in clips]
        self.noise = torch.cat([p.to(core.device) for p in parts] + [torch.zeros(0, dtype=torch.int16, device=core.device)])
        if self.noise.numel() == 0:
            raise ValueError('the noise corpus is empty')
        if not 0 <= int(pos) < self.noise.numel():
            raise ValueError('pos = %d outside [0, %d)' % (int(pos), self.noise.numel()))
        self.pos = int(pos)

    def __len__(self):
        return int(self.noise.numel())


def _noise_calls(core: PreciseB200, clips, items):
    """The library calls of a mix over items[i] = clip index, split as vectorize_clips splits clips: a list of (packed pcm,
    offsets, the items' entries, first item, item count, samples)."""
    clips = [_check_recording(core, c) for c in clips]
    items = np.arange(len(clips), dtype=np.int64) if items is None else np.asarray(items, np.int64)
    if items.ndim != 1:
        raise ValueError('items must be a 1-D array')
    if items.size and (items.min() < 0 or items.max() >= len(clips)):
        raise ValueError('items must lie in [0, %d)' % len(clips))
    calls, first = [], 0
    for g in _call_groups([clips[i] for i in items]) if items.size else []:
        uniq, local = np.unique(items[first:first + len(g)], return_inverse=True)
        pcm, offsets, entry = _pack(core, [clips[i] for i in uniq])
        calls.append((pcm, offsets, entry[local].astype(np.int32), first, len(g), sum(int(c.shape[0]) for c in g)))
        first += len(g)
    return calls, int(items.size)


def _mix_calls(core: PreciseB200, calls, n_items, noise, pos, ratios, out, inputs):
    """pb_add_noise over _noise_calls' calls, the noise position carried from call to call.  Returns (int16 tensor or None,
    float32 tensor or None, position after the last item)."""
    torch = core.torch
    ratios = np.asarray(ratios, np.float64)
    if ratios.shape != (n_items,):
        raise ValueError('one ratio per item')
    outs, ins = [], []
    for pcm, offsets, entries, first, count, samples in calls:
        o, x = core.add_noise(pcm, offsets, noise, entries, ratios[first:first + count], pos, out=out, inputs=inputs)
        outs.append(o)
        ins.append(x)
        pos = (pos + samples) % int(noise.numel())
    cat = lambda parts, empty: (parts[0] if len(parts) == 1 else torch.cat(parts)) if parts else empty
    o = cat(outs, torch.zeros(0, dtype=torch.int16, device=core.device)) if out else None
    x = cat(ins, torch.empty((0, core.n_features, core.feature_size), dtype=torch.float32, device=core.device)) if inputs else None
    return o, x, pos


def _mix_groups(core: PreciseB200, clips, noise, pos, ratios, items, out, inputs):
    calls, n_items = _noise_calls(core, clips, items)
    return _mix_calls(core, calls, n_items, noise, pos, ratios, out, inputs)


def add_noise(core: PreciseB200, clips, source: NoiseSource, ratios, items=None):
    """precise-add-noise's noised_audio on the device: item i is clips[items[i]] (items None: every clip once, in order)
    mixed with the next stretch of ``source``'s noise at ratio ratios[i] (pb_add_noise's arithmetic; the reference's
    differences are a silent span adding no noise and out-of-range values saturating).  Clips are 1-D int16 numpy arrays or
    CUDA tensors read as load_audio reads them; empty ones give empty clips.  Returns (int16 CUDA tensor of the mixed clips
    back to back, host int64 offsets [n_items + 1]) and advances source.pos; one call or many give the same clips."""
    n = len(clips) if items is None else len(items)
    lens = np.asarray([int(clips[i].shape[0]) for i in (range(n) if items is None else items)], np.int64)
    o, _, source.pos = _mix_groups(core, clips, source.noise, source.pos, ratios, items, True, False)
    return o, np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)


def vectorize_noisy(core: PreciseB200, clips, source: NoiseSource, ratios, items=None):
    """vectorize of each of add_noise's clips (none may be empty), float32 [n_items, n_features, feature_size], without the
    mixed clips leaving the device: the rows pb_vectorize_clips makes of them when each clip's last max_samples samples start
    at a multiple of 8 samples (so with the generic K1 forced, bit for bit vectorize_clips(add_noise(...))).  Advances
    source.pos as add_noise does."""
    _, x, source.pos = _mix_groups(core, clips, source.noise, source.pos, ratios, items, False, True)
    return x


_M64 = (1 << 64) - 1


def _mix64(z):
    """splitmix64's finalizer (pb_train's key, include/precise_b200.h)."""
    z &= _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def _key(s, e, j, c):
    return _mix64(_mix64(_mix64(_mix64(s) + e) + j) + c)


@dataclass
class Augment:
    """Noise augmentation of a training run (train's ``augment``): in every epoch each clip gets ``copies`` fresh noisy
    copies from ``source``.  In epoch e, item i (clip i // copies, copy i % copies) has ratio low + (high - low) u with
    u = (key(seed, e, i, 0) >> 11) 2^-53, and the epoch's noise starts at (source.pos + e * copies * sum of the clip lengths)
    mod len(source); source.pos itself is not moved.  So a resumed fit draws exactly the noise of an uninterrupted one."""
    source: NoiseSource
    copies: int = 1
    low: float = 0.0
    high: float = 0.4
    seed: int = 0

    def ratios(self, epoch, n_items):
        u = np.asarray([(_key(int(self.seed), int(epoch), i, 0) >> 11) * 2.0 ** -53 for i in range(n_items)], np.float64)
        return self.low + (self.high - self.low) * u

    def position(self, epoch, clip_samples):
        return (self.source.pos + int(epoch) * self.copies * int(clip_samples)) % len(self.source)


def _train_augmented(core, state, clips, targets, rows, recs, epochs, kw, augment: Augment, validation_step):
    """train with augment: one pb_train call per epoch over the clean clips plus each clip's noisy copies, clip-major."""
    torch = core.torch
    M = int(augment.copies)
    if M < 1:
        raise ValueError('copies must be >= 1')
    clips = [_check_recording(core, c) for c in clips]
    n = len(clips)
    targets = np.asarray(targets)
    if targets.shape != (n,):
        raise ValueError('one target per clip')
    clean = vectorize_clips(core, clips)
    items = np.repeat(np.arange(n, dtype=np.int64), M)
    calls, _ = _noise_calls(core, clips, items)                # packed once, mixed afresh every epoch
    samples = sum(int(c.shape[0]) for c in clips)
    tg = np.repeat(targets != 0, M + 1).astype(np.uint8)
    if rows is not None:
        rows = np.repeat(np.asarray(rows, np.int32), M + 1)
        recs = (np.repeat(np.asarray(recs, np.int64), M + 1) * (M + 1) + np.tile(np.arange(M + 1), len(recs))).astype(np.int64)
        kw = dict(kw, rows_of=rows, recs=recs)
    losses = []
    for _ in range(epochs):
        e = state.epoch
        _, noisy, _ = _mix_calls(core, calls, n * M, augment.source.noise, augment.position(e, samples),
                                 augment.ratios(e, n * M), False, True)
        x = torch.empty((n, M + 1, core.n_features, core.feature_size), dtype=torch.float32, device=core.device)
        x[:, 0] = clean
        x[:, 1:] = noisy.view(n, M, core.n_features, core.feature_size)
        x = x.view(n * (M + 1), core.n_features, core.feature_size)
        losses.append(core.train(x, tg, state.rows, state.weights, state.rms, epochs=1, epoch0=e, **kw))
        state.epoch += 1
        validation_step()
    k = len(state.hidden)
    return core.torch.cat(losses, 1).cpu().numpy() if losses else np.zeros((k, 0))


# ---- generated training audio (precise-train-generated) ----------------------------------------------------------------------

# Samples per pb_generate call of Generator.run (items are never split: a longer item is a call of its own).  At the cap a
# call's device memory stays under 256 MB: d_out and the aligned workspace 64 MB each (int16), the frame rows about 3 MB
# at the default hop, and the chosen windows' inputs at most 25 MB (one 1 508-byte window per 2 048-sample chunk).
GENERATE_CALL_SAMPLES = 1 << 25

# Window-less items in a row after which Generator gives up rather than loop: the label rule keeps the window at the end of
# any silence longer than the label buffer, so this takes a buffer longer than the longest silence (2.5 s).
_GENERATE_IDLE = 10000


def _unit(seed, e, j, c):
    """A uniform double in [0, 1) from pb_train's splitmix key: (key(s, e, j, c) >> 11) 2^-53."""
    return (_key(int(seed), int(e), int(j), int(c)) >> 11) * 2.0 ** -53


class _LabelTail:
    """vals_buffer (train_generated.py:176): the last ``n`` per-sample labels of the whole run, kept as the runs of ones
    [a, b) of the label stream, which starts with n zeros.  ``end`` is the stream's length so far."""

    def __init__(self, n):
        self.n, self.end, self.runs = int(n), int(n), []

    def add(self, length, one):
        if one and length > 0:
            if self.runs and self.runs[-1][1] == self.end:
                self.runs[-1][1] += length
            else:
                self.runs.append([self.end, self.end + length])
        self.end += length

    def decide(self, p):
        """The label rule of the window whose buffer ends at stream position p (no earlier than the last call's):
        1, 0, or -1 for a skipped window."""
        lo = p - self.n
        while self.runs and self.runs[0][1] <= lo:
            self.runs.pop(0)
        best, last = 0, 0
        for a, b in self.runs:
            if a >= p:
                break
            best = max(best, min(b, p) - max(a, lo))
            last = b >= p
        frac = best / self.n
        if not last and frac > 0.8:
            return 1
        return 0 if frac < 0.5 else -1

    def copy(self):
        t = _LabelTail(self.n)
        t.end, t.runs = self.end, [list(r) for r in self.runs]
        return t


@dataclass
class GeneratedItem:
    """One background file's pass: background b at gain f, the first ``length`` samples generated, its segments
    [(clip or -1, first sample, samples)] and its windows [(chunk index, target)] (skipped chunks left out)."""
    background: int
    f: float
    length: int
    segments: list
    windows: list


class Generator:
    """precise-train-generated's sample generator (train_generated.py:118-213) with keyed randomness.

    Backgrounds are taken in the order of (key(seed, 0, b, 0), b), cycled forever; pass p's item of background b draws
    u_c = (key(seed, p + 1, b, c) >> 11) 2^-53 (pb_train's key): c = 0 the volume, f = 0.4 + 0.5 u_0; then the wake-word
    pieces, piece k drawing u_{1 + k}: a clip (even k; a wake word if u > 0.5, the next of the wake_clips cycle, else the next
    of other_clips) or a silence of int(sample_rate (0.5 + 2 u)) samples (odd k).  Pieces are drawn only as the chunks need
    them, as the reference's generators draw them.  The stream is cut as chunk_audio_pieces cuts it (each ``combined`` the
    previous piece followed by the current one: DESIGN §3 "Generated training audio"), and chunk c's window is labelled by vals_buffer's rule
    (a run of ones over 0.8 of buffer_samples ending before the last sample: 1; under 0.5: 0; else skipped).  The clip
    cycles and the label tail carry over items, passes and epochs, as in the reference.

    plan(n) takes the next n windows; an item cut at the end of a plan continues in the next one (its stream is generated
    again from its start).  at(epoch, entries) replays the plan, so a resumed run draws what an uninterrupted one would.
    core None: plans only (no device data)."""

    def __init__(self, core, backgrounds, wake_clips, other_clips, chunk=2048, seed=0, names=None, sample_rate=None,
                 buffer_samples=None):
        if not len(wake_clips) or not len(other_clips):
            raise ValueError('the generator needs at least one wake-word and one not-wake-word clip')
        if not len(backgrounds):
            raise ValueError('the generator needs at least one background recording')
        self.core, self.chunk, self.seed = core, int(chunk), int(seed)
        if self.chunk < 1:
            raise ValueError('chunk must be >= 1')
        pr = core.params if core is not None else None
        self.sample_rate = int(sample_rate if sample_rate is not None else pr.sample_rate)
        self.buffer_samples = int(buffer_samples if buffer_samples is not None else pr.buffer_samples)
        self.bg_lens = [int(b.shape[0]) for b in backgrounds]
        if max(self.bg_lens) <= self.chunk:
            raise ValueError('every background is at most one chunk (%d samples) long: none gives a window' % self.chunk)
        self.clip_lens = [int(c.shape[0]) for c in list(wake_clips) + list(other_clips)]
        self.n_wake, self.n_other = len(wake_clips), len(other_clips)
        self.names = list(names) if names is not None else ['%d' % b for b in range(len(backgrounds))]
        self.order = sorted(range(len(backgrounds)), key=lambda b: (_key(self.seed, 0, b, 0), b))
        self._dev = None
        if core is not None:
            torch = core.torch
            cat = lambda recs: torch.cat([torch.as_tensor(_check_recording(core, r)).to(core.device) for r in recs]
                                         + [torch.zeros(0, dtype=torch.int16, device=core.device)])
            offs = lambda lens: np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
            self._dev = (cat(backgrounds), offs(self.bg_lens), cat(list(wake_clips) + list(other_clips)), offs(self.clip_lens))
        self._reset()

    def _reset(self):
        self.taken = 0                                        # windows planned so far
        self.pass_, self.q = 0, 0                             # the next item: order[q] of pass pass_
        self.next_wake = self.next_other = 0
        self.tail = _LabelTail(self.buffer_samples)
        self.cur, self.cur_w = None, 0                        # the item being taken and its windows taken
        self.idle = 0                                         # items in a row without a window

    def _item(self, p, b):
        ch, seed = self.chunk, self.seed
        n = max(0, (self.bg_lens[b] - 1) // ch)              # len(range(chunk, len, chunk))
        f = 0.4 + 0.5 * _unit(seed, p + 1, b, 0)
        start = self.tail.end
        segs, need, got, prev, k = [], n * ch, 0, None, 0
        while got < need:
            u = _unit(seed, p + 1, b, 1 + k)
            if k % 2 == 0:
                wake = u > 0.5
                if wake:
                    piece = (self.next_wake, self.clip_lens[self.next_wake], True)
                    self.next_wake = (self.next_wake + 1) % self.n_wake
                else:
                    c = self.n_wake + self.next_other
                    piece = (c, self.clip_lens[c], False)
                    self.next_other = (self.next_other + 1) % self.n_other
            else:
                piece = (-1, int(self.sample_rate * (0.5 + 2.0 * u)), False)
            both = [piece] if prev is None or prev[1] == 0 else [prev, piece]
            total = sum(x[1] for x in both)
            rem = min(((total - 1) // ch if total > 0 else 0) * ch, need - got)
            got += rem
            for clip, length, wake in both:
                m = min(length, rem)
                if m > 0:
                    segs.append((clip, 0, m))
                    self.tail.add(m, wake)
                rem -= m
            prev, k = piece, k + 1
        windows = []
        for c in range(n):
            t = self.tail.decide(start + (c + 1) * ch)
            if t >= 0:
                windows.append((c, t))
        return GeneratedItem(b, f, n * ch, segs, windows)

    def _next_item(self):
        b = self.order[self.q]
        item = self._item(self.pass_, b)
        self.q += 1
        if self.q == len(self.order):
            self.q, self.pass_ = 0, self.pass_ + 1
        self.idle = 0 if item.windows else self.idle + 1
        if self.idle > _GENERATE_IDLE:
            raise ValueError('the label rule skipped every window of %d items in a row' % _GENERATE_IDLE)
        return item

    def plan(self, n):
        """The next n windows: a list of (GeneratedItem, first window, end window)."""
        out, left = [], int(n)
        while left > 0:
            if self.cur is None or self.cur_w == len(self.cur.windows):
                self.cur, self.cur_w = self._next_item(), 0
            take = min(left, len(self.cur.windows) - self.cur_w)
            if take:
                out.append((self.cur, self.cur_w, self.cur_w + take))
            self.cur_w += take
            left -= take
        self.taken += int(n)
        return out

    def seek(self, windows):
        """Moves to the state after ``windows`` windows have been planned (replaying from the start if needed)."""
        windows = int(windows)
        if windows < self.taken:
            self._reset()
        if windows > self.taken:
            self.plan(windows - self.taken)
        return self

    def at(self, epoch, entries):
        """A copy of this generator at the start of ``epoch`` of ``entries`` windows per epoch."""
        g = object.__new__(Generator)
        g.__dict__.update(self.__dict__)
        g._reset()
        return g.seek(int(epoch) * int(entries))

    def tables(self, plan):
        """pb_generate's tables of a plan: (GEN_ITEM items, GEN_SEGMENT segments, int64 windows [n, 2], uint8 targets)."""
        from .core import GEN_ITEM, GEN_SEGMENT
        items = np.zeros(len(plan), GEN_ITEM)
        segs, wins, tg = [], [], []
        for i, (it, w0, w1) in enumerate(plan):
            chosen = it.windows[w0:w1]
            length = (chosen[-1][0] + 1) * self.chunk
            s0 = len(segs)
            cover = 0
            for s in it.segments:
                if cover >= length:
                    break
                segs.append(s)
                cover += s[2]
            items[i] = (it.background, 0, it.f, length, s0, len(segs))
            wins += [(i, c) for c, _ in chosen]
            tg += [t for _, t in chosen]
        seg = np.zeros(len(segs), GEN_SEGMENT)
        for j, (c, a, m) in enumerate(segs):
            seg[j] = (c, 0, a, m)
        return items, seg, np.asarray(wins, np.int64).reshape(-1, 2), np.asarray(tg, np.uint8)

    def run(self, plan, out=False, divisor=32767):
        """pb_generate over a plan, in calls of at most GENERATE_CALL_SAMPLES samples: (network inputs float32
        [n, n_features, feature_size], targets uint8 [n], and with out=True the streams (int16 tensor) with each window's
        end sample in them, int64 [n]; else None, None)."""
        core = self.core
        torch = core.torch
        bg, bg_off, clips, clip_off = self._dev
        groups, cur, size = [], [], 0
        for p in plan:
            L = (p[0].windows[p[2] - 1][0] + 1) * self.chunk
            if cur and size + L > GENERATE_CALL_SAMPLES:
                groups.append(cur)
                cur, size = [], 0
            cur.append(p)
            size += L
        if cur:
            groups.append(cur)
        ins, tgs, outs, ends, base = [], [], [], [], 0
        for g in groups:
            items, seg, wins, tg = self.tables(g)
            o, x = core.generate(bg, bg_off, clips, clip_off, items, seg, wins, self.chunk, divisor, out=out)
            ins.append(x)
            tgs.append(tg)
            if out:
                starts = base + np.concatenate([[0], np.cumsum(items['length'])])[wins[:, 0]]
                ends.append(starts + (wins[:, 1] + 1) * self.chunk)
                outs.append(o)
                base += int(items['length'].sum())
        empty = torch.empty((0, core.n_features, core.feature_size), dtype=torch.float32, device=core.device)
        x = (ins[0] if len(ins) == 1 else torch.cat(ins)) if ins else empty
        tg = np.concatenate(tgs) if tgs else np.zeros(0, np.uint8)
        if not out:
            return x, tg, None, None
        audio = torch.cat(outs) if outs else torch.zeros(0, dtype=torch.int16, device=core.device)
        return x, tg, audio, (np.concatenate(ends) if ends else np.zeros(0, np.int64))


def _save_generated(gen, epoch, plan, audio, ends, targets, save_prob, folder):
    """-p: entry j of the epoch is saved when (key(seed, epoch, j, 2^32) >> 11) 2^-53 > 1 - save_prob, as
    debug/{ww,nww}/'<background> - <chunk>.wav': the buffer_samples generated samples that end at its window (zeros before
    its background's stream starts)."""
    import os
    from .add_noise import write_wav
    B = gen.buffer_samples
    a = audio.cpu().numpy()
    j = 0
    for it, w0, w1 in plan:
        for c, t in it.windows[w0:w1]:
            if _unit(gen.seed, epoch, j, 1 << 32) > 1.0 - save_prob:
                e = int(ends[j])
                s = max(e - B, e - (c + 1) * gen.chunk)
                buf = np.zeros(B, np.int16)
                buf[B - (e - s):] = a[s:e]
                name = '%s - %d.wav' % (os.path.splitext(os.path.basename(gen.names[it.background]))[0], c)
                write_wav(os.path.join(folder, 'ww' if targets[j] else 'nww', name), buf, gen.sample_rate)
            j += 1


def train_generated(core: PreciseB200, state: TrainState, gen: Generator, epochs, steps_per_epoch=100, batch_size=200,
                    sensitivity=0.2, dropout=0.2, validation=None, save_prob=0.0, debug_folder='debug'):
    """precise-train-generated's fit_generator for every network of ``state`` at once: each epoch is the generator's next
    steps_per_epoch x batch_size windows (Generator.run: pb_generate) and one pb_train epoch over them with
    epoch0 = state.epoch, every network on the same entries.  The generator is first moved to epoch state.epoch, so a
    resumed run trains on what an uninterrupted one would.  pb_train shuffles the entries where fit_generator takes
    consecutive batches.  Returns the epoch losses [k, epochs]; with validation=(inputs, targets) also val_loss
    (pb_train_loss, as train's).  save_prob > 0 writes debug wavs of the chosen windows (_save_generated)."""
    n = int(steps_per_epoch) * int(batch_size)
    if n < 1:
        raise ValueError('steps_per_epoch and batch_size must be >= 1')
    lb = 1.0 - sensitivity
    losses, vals = [], []
    for _ in range(int(epochs)):
        e = state.epoch
        gen.seek(e * n)
        plan = gen.plan(n)
        x, tg, audio, ends = gen.run(plan, out=save_prob > 0)
        losses.append(core.train(x, tg, state.rows, state.weights, state.rms, epochs=1, epoch0=e, batch_size=batch_size,
                                 loss_bias=lb, dropout=dropout))
        state.epoch += 1
        if validation is not None:
            vals.append(core.train_loss(validation[0], validation[1], state.rows, state.weights, loss_bias=lb))
        if save_prob > 0:
            _save_generated(gen, e, plan, audio, ends, tg, save_prob, debug_folder)
    k = len(state.hidden)
    loss = core.torch.cat(losses, 1).cpu().numpy() if losses else np.zeros((k, 0))
    if validation is None:
        return loss
    return loss, core.torch.stack(vals, 1).cpu().numpy() if vals else np.zeros((k, 0))
