"""Many independent audio streams per call -- the throughput path (no reference equivalent: the
reference runs one Listener per process).  Semantically ``S`` x [Listener.update ->
TriggerDetector.update] per tick, all state device-resident.
"""
import numpy as np

from .core import PreciseB200
from .model_io import GruModel
from .params import ListenerParams


class StreamBatch:
    def __init__(self, model: GruModel, n_streams: int, params: ListenerParams = None, chunk_samples=1024,
                 device=0, sensitivity=0.5, trigger_level=3):
        self.pr = params or ListenerParams()
        self.n_streams = n_streams
        self.core = PreciseB200(self.pr, hidden=model.hidden, max_streams=n_streams, chunk_samples=chunk_samples,
                                device=device, sensitivity=sensitivity, trigger_level=trigger_level,
                                activation=model.activation, recurrent_activation=model.recurrent_activation)
        self.core.load_weights(model.kernel, model.recurrent, model.bias, model.dense_w, model.dense_b)
        torch = self.core.torch
        self.count = torch.zeros(1, dtype=torch.int64, device=self.core.device)
        self.counts = torch.zeros(1, dtype=torch.int64, device=self.core.device)    # per bank model, update_models / update_ragged
        self._out = None
        self._bank_out = None

    def add_model(self, model, params: ListenerParams = None, sensitivity=0.5, trigger_level=3, decode_legacy_f64=False) -> int:
        """Score another network (GruModel or weights path) on the same streams' MFCC frames; returns its bank slot.
        See PreciseB200.add_model."""
        slot = self.core.add_model(model, params, sensitivity, trigger_level, decode_legacy_f64)
        torch = self.core.torch
        self.counts = torch.cat([self.counts, torch.zeros(1, dtype=torch.int64, device=self.core.device)])
        self._bank_out = None
        return slot

    def set_stream_models(self, masks, ids=None):
        """Which bank models score which streams: bit m of masks[i] (host uint8) = slot m scores stream ids[i] (host int32;
        None: stream i).  Unsubscribed pairs come back as NaN / NaN / 0.  See PreciseB200.set_stream_models."""
        self.core.set_stream_models(masks, ids)

    def set_stream_trigger(self, slot, sensitivity, trigger_level, chunk_size, ids=None):
        """Each stream's TriggerDetector(chunk_size in bytes, sensitivity, trigger_level) for bank slot ``slot``; scalars
        broadcast.  See PreciseB200.set_stream_trigger."""
        self.core.set_stream_trigger(slot, sensitivity, trigger_level, chunk_size, ids)

    def stream_trigger(self, slot, ids=None):
        """(sensitivity, trigger_level, chunk_size) host arrays of bank slot ``slot``.  See PreciseB200.stream_trigger."""
        return self.core.stream_trigger(slot, ids)

    def _bank_buffers(self, n):
        """The cached [M, n] outputs of a bank tick."""
        M = self.core.num_models
        if self._bank_out is None or tuple(self._bank_out['conf'].shape) != (M, n):
            torch = self.core.torch
            dev = self.core.device
            self._bank_out = dict(raw=torch.empty((M, n), dtype=torch.float32, device=dev),
                                  conf=torch.empty((M, n), dtype=torch.float64, device=dev),
                                  fired=torch.empty((M, n), dtype=torch.uint8, device=dev))
        return self._bank_out

    def update_models(self, pcm, ids=None):
        """One tick for every bank model: pcm int16 CUDA [n, chunk_samples] -> dict(raw f32, conf f64, fired u8), each
        [M, n].  ``self.counts`` (int64[M], device) accumulates each model's fired streams until reset_count()."""
        return self.core.update_models(pcm, ids, self._bank_buffers(pcm.shape[0]), self.counts)

    def update_ragged(self, pcm, offsets, ids=None, max_len=None):
        """Ragged tick for every bank model: stream item i brings pcm[offsets[i]:offsets[i + 1]] (1-D int16 CUDA pcm, int64
        CUDA offsets [n + 1]) -> dict(raw, conf, fired), each [M, n], accumulating ``self.counts``.  See
        PreciseB200.update_ragged."""
        return self.core.update_ragged(pcm, offsets, ids, max_len, self._bank_buffers(offsets.numel() - 1), self.counts)

    def update(self, pcm, ids=None):
        """pcm: int16 CUDA tensor [n, chunk_samples] -> dict(raw f32[n], conf f64[n], fired u8[n]).
        ``self.count`` (int64[1], device) accumulates fired streams until reset_count()."""
        n = pcm.shape[0]
        if self._out is None or self._out['conf'].shape[0] != n:
            torch = self.core.torch
            dev = self.core.device
            self._out = dict(raw=torch.empty(n, dtype=torch.float32, device=dev),
                             conf=torch.empty(n, dtype=torch.float64, device=dev),
                             fired=torch.empty(n, dtype=torch.uint8, device=dev))
        return self.core.update(pcm, ids, self._out, self.count)

    def update_host(self, pcm_np: np.ndarray, conf_np: np.ndarray, raw_np=None, fired_np=None) -> int:
        return self.core.update_host(pcm_np, conf_np, raw_np, fired_np)

    def reset_count(self):
        self.count.zero_()
        self.counts.zero_()

    def clear(self, ids=None):
        self.core.clear(ids=ids) if ids is not None else self.core.clear()
