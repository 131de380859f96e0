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

Training (fused-family networks, many per call: pb_vectorize_clips, pb_train, pb_train_loss):
  vectorize_clips   vectorize(clip) of every clip, on the device
  TrainState, train ~ precise/model.py:57-91, scripts/train.py:159-166 (Keras fit: loss, dropout, RMSprop; val_loss)
"""
from dataclasses import dataclass

import numpy as np

from .core import PB_TRAIN_STRIDE, PreciseB200, threshold_encode
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
    [k, PB_TRAIN_STRIDE] (Keras's order: kernel, recurrent, bias, dense_w, dense_b), each row's hidden size, activations and
    seed, and the next epoch's number (the shuffles and dropout masks of a resumed fit continue from it)."""

    def __init__(self, core: PreciseB200, weights, rms, hidden, activation, recurrent_activation, seeds, epoch=0):
        self.core = core
        self.weights, self.rms = weights, rms
        self.hidden, self.activation, self.recurrent_activation = list(hidden), list(activation), list(recurrent_activation)
        self.seeds = [int(s) for s in seeds]
        self.epoch = int(epoch)
        self.rows = core.train_rows(self.hidden, self.activation, self.recurrent_activation, self.seeds)

    @staticmethod
    def from_models(core: PreciseB200, models, seeds):
        """One row per GruModel (feature size core.feature_size, hidden <= 24), accumulators at zero."""
        torch = core.torch
        w = np.zeros((len(models), PB_TRAIN_STRIDE), np.float32)
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


def train(core: PreciseB200, state: TrainState, inputs, targets, rows=None, recs=None, epochs=10, batch_size=5000,
          sensitivity=0.2, dropout=0.2, lr=0.001, validation=None):
    """precise-train's fit for every network of ``state`` at once (pb_train): ``epochs`` epochs over ``inputs``
    (vectorize_clips' tensor) with labels ``targets`` (non-zero = wake word), loss_bias = 1 - sensitivity (train.py:86).
    rows / recs None: every network on every input; otherwise entry p is inputs[recs[p]] for network rows[p] (each word
    on its owner's clips plus shared negatives).  state.epoch advances by ``epochs``.  Returns the epoch losses, float64
    [k, epochs]; with validation=(inputs, targets) or (inputs, targets, rows, recs) also val_loss [k, epochs], each
    network's loss over its validation entries without dropout after each epoch (pb_train_loss, Keras's evaluate)."""
    kw = dict(rows_of=rows, recs=recs, batch_size=batch_size, lr=lr, loss_bias=1.0 - sensitivity, dropout=dropout)
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
