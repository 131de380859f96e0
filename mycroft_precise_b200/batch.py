"""Many independent audio streams per call -- the throughput path (no reference equivalent: the
reference runs one Listener per process).  Semantically ``S`` x [Listener.update ->
TriggerDetector.update] per tick, all state device-resident.
"""
import numpy as np

from .core import FRONT_END_FIELDS, PreciseB200, _check_np
from .model_io import GruModel
from .params import ListenerParams

STATE_FIELDS = ('magic', 'version', 'num_models') + FRONT_END_FIELDS    # the first 12 int32 words of a state record


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
        self.pool_count = torch.zeros(1, dtype=torch.int64, device=self.core.device)   # pool fires, update_pool
        self._out = None
        self._bank_out = None
        self._pool_specs = {}                # pool slot -> pool_load's arguments, for pool_calibrate

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

    def set_pool(self, max_models):
        """A model pool of ``max_models`` slots beside the bank; each stream is scored by at most one pool model.  See
        PreciseB200.set_pool."""
        self.core.set_pool(max_models)
        self._pool_specs = {}

    def pool_load(self, model_id, model, params: ListenerParams = None, sensitivity=0.5, trigger_level=3, decode_legacy_f64=False):
        """Load a network (GruModel or weights path) into pool slot ``model_id``.  See PreciseB200.pool_load."""
        self.core.pool_load(model_id, model, params, sensitivity, trigger_level, decode_legacy_f64)
        self._pool_specs[int(model_id)] = (model, params, sensitivity, trigger_level, decode_legacy_f64)

    def pool_calibrate(self, model_ids, clips, rows=None, recs=None, smoothing=1.2):
        """precise-calc-threshold for pool slots ``model_ids`` (int32 [k], loaded through this batch's pool_load) from
        wake-word clips: entry p is model_ids[rows[p]] over clips[recs[p]], each word over its owner's recordings (rows /
        recs None: every model over every clip).  Each slot whose clips give a fit is loaded again with
        threshold_config ((mu, std),) through pool_load, which re-arms its streams as a newly loaded model does; a slot
        without data keeps its table.  Returns the list of k fits, (mu, std) or None.  See offline.calc_threshold."""
        from .offline import calc_threshold, test_pool
        from .runner import _resolve_model
        specs = [self._pool_specs[int(m)] for m in model_ids]
        stats = test_pool(self.core, clips, np.ones(len(clips), np.uint8), model_ids, rows, recs)
        fits = [calc_threshold(st, smoothing) for st in stats]
        for mid, fit, (model, params, sens, lvl, legacy) in zip(model_ids, fits, specs):
            if fit is None:
                continue
            base = params or _resolve_model(model)[1] or self.pr
            pr = ListenerParams(**dict(base.to_dict(), threshold_config=(fit,)))
            self.pool_load(int(mid), model, pr, sens, lvl, legacy)
        return fits

    def pool_train(self, model_ids, models, clips, targets, rows=None, recs=None, seeds=None, **opts):
        """precise-train for pool slots ``model_ids`` (int32 [k]) starting from ``models`` (k GruModels, e.g. the slots'
        current networks or GruModel.init), on labelled ``clips`` (1-D int16, read as load_audio reads them; targets non-zero =
        wake word): rows / recs as offline.train takes them, ``opts`` its keyword arguments, seeds [k] (default 0 .. k-1).
        Each trained network is loaded into its slot through pool_load with the slot's earlier settings (those of this batch's
        pool_load, or the defaults), which re-arms its streams as a newly loaded model does.  Returns the k trained GruModels."""
        from .offline import TrainState, train, vectorize_clips
        from .runner import _resolve_model
        inputs = vectorize_clips(self.core, clips)
        state = TrainState.from_models(self.core, models, range(len(models)) if seeds is None else seeds)
        train(self.core, state, inputs, targets, rows, recs, **opts)
        out = state.models()
        for mid, m in zip(model_ids, out):
            spec = self._pool_specs.get(int(mid))
            if spec is None:
                self.pool_load(int(mid), m)
                continue
            model, params, sens, lvl, legacy = spec
            self.pool_load(int(mid), m, params or _resolve_model(model)[1] or self.pr, sens, lvl, legacy)
        return out

    def set_stream_pool(self, model_ids, ids=None):
        """Each stream's pool model (host int32, -1 = none).  See PreciseB200.set_stream_pool."""
        self.core.set_stream_pool(model_ids, ids)

    def stream_pool(self, ids=None):
        """Host int32 array: each stream's pool model, -1 = none.  See PreciseB200.stream_pool."""
        return self.core.stream_pool(ids)

    def update_pool(self, pcm, ids=None, offsets=None, max_len=None):
        """One pool tick (update's with pcm [n, chunk_samples]; update_ragged's with 1-D pcm and ``offsets``) -> dict(raw,
        conf, fired), each [n].  ``self.pool_count`` accumulates pool fires until reset_count().  See
        PreciseB200.update_pool."""
        return self.core.update_pool(pcm, ids, offsets, max_len, count=self.pool_count)

    def update_all(self, pcm, ids=None, offsets=None, max_len=None):
        """One combined tick, the bank and the pool on one K1 (uniform with pcm [n, chunk_samples], ragged with 1-D pcm and
        ``offsets``) -> dict(raw, conf, fired), each [M + 1, n]: rows 0 .. M-1 as update_models / update_ragged, row M as
        update_pool.  Accumulates ``self.counts`` and ``self.pool_count``.  See PreciseB200.update_all."""
        return self.core.update_all(pcm, ids, offsets, max_len, counts=self.counts, pool_count=self.pool_count)

    def set_stream_pool_trigger(self, sensitivity, trigger_level, chunk_size, ids=None):
        """Each stream's TriggerDetector(chunk_size in bytes, sensitivity, trigger_level) on its pool model; chunk_size 0 =
        the model's own settings; scalars broadcast.  See PreciseB200.set_stream_pool_trigger."""
        self.core.set_stream_pool_trigger(sensitivity, trigger_level, chunk_size, ids)

    def stream_pool_trigger(self, ids=None):
        """(sensitivity, trigger_level, chunk_size) host arrays of the streams' pool settings; (NaN, 0, 0) = the model's own.
        See PreciseB200.stream_pool_trigger."""
        return self.core.stream_pool_trigger(ids)

    def set_history(self, samples=None, max_rows=None):
        """A device pool for the recent audio of up to ``max_rows`` streams, ``samples`` each (default buffer_samples, the
        reference's clip).  See PreciseB200.set_history."""
        self.core.set_history(samples, max_rows)

    def set_stream_history(self, on, ids=None):
        """Switch each stream's history on or off; a scalar broadcasts.  See PreciseB200.set_stream_history."""
        self.core.set_stream_history(on, ids)

    def stream_history(self, ids=None):
        """Host bool array: which streams have history.  See PreciseB200.stream_history."""
        return self.core.stream_history(ids)

    def read_history(self, ids=None, samples=None, out=None):
        """int16 CUDA [n, samples]: each stream's last samples, oldest first.  See PreciseB200.read_history."""
        return self.core.read_history(ids, samples, out)

    def activation_audio(self, fired, ids=None, samples=None):
        """The clip behind every activation of the tick just run, as listen.py saves it in on_activation: ``fired`` and ``ids``
        are that tick's output ([n] or [M, n]) and ids (int32 CUDA tensor; None: items are streams 0..n-1).  Returns dict(slot =
        bank slot, stream = stream id, audio = int16 [k, samples] ending with that tick's chunk) for every fired (model, item)
        pair whose stream has history, in torch.nonzero order (model-major).  On update_all's [M + 1, n] output, slot == M
        means the stream's pool model.  Call it before the next tick on those streams."""
        core = self.core
        torch = core.torch
        f = fired if fired.dim() == 2 else fired.reshape(1, -1)
        n = f.shape[1]
        if ids is None:
            ids = torch.arange(n, dtype=torch.int32, device=core.device)
        core._check_t('ids', ids, torch.int32, n, optional=False)
        pairs = torch.nonzero(f)
        streams = ids[pairs[:, 1]]
        # a stream that fired on several rows appears once per row: look it up and read its clip once
        uniq, inv = torch.unique(streams, return_inverse=True)
        has = torch.from_numpy(core.stream_history(uniq.cpu().numpy().astype(np.int32))).to(core.device)
        keep = has[inv]
        pairs, streams = pairs[keep], streams[keep].contiguous()
        if streams.numel() == 0:
            s = core.history_samples if samples is None else int(samples)
            audio = torch.empty((0, s), dtype=torch.int16, device=core.device)
        else:
            uniq, inv = torch.unique(streams, return_inverse=True)
            audio = core.read_history(uniq.contiguous(), samples)[inv]
        return dict(slot=pairs[:, 0], stream=streams, audio=audio)

    def _host_ids(self, ids, n):
        _check_np('ids', ids, np.int32, (n,))
        if ids is None:
            return np.arange(n, dtype=np.int32)
        if n and (ids.min() < 0 or ids.max() >= self.n_streams or len(np.unique(ids)) != n):
            raise ValueError('stream ids must be unique and lie in [0, %d)' % self.n_streams)
        return ids

    def export_streams(self, ids=None):
        """A snapshot of streams ids (host int32 array; None: every stream): dict(state = their state records, a uint8 CUDA
        tensor [n, stream_state_bytes]; stream_models = their masks; stream_trigger = each bank slot's (sensitivity,
        trigger_level, chunk_size); with a model pool, stream_pool = their pool models and stream_pool_trigger = their pool
        (sensitivity, trigger_level, chunk_size)).  The tensor may go through .cpu() or
        .to(another device) and come back.  Whether a stream has audio history, and that audio, are not part of a snapshot.
        See PreciseB200.export_streams."""
        core = self.core
        n = self.n_streams if ids is None else (ids.shape[0] if isinstance(ids, np.ndarray) and ids.ndim == 1 else -1)
        sids = self._host_ids(ids, n)
        state = core.export_streams(core.torch.from_numpy(sids).to(core.device))
        snap = dict(state=state, stream_models=core.stream_models(sids),
                    stream_trigger=[core.stream_trigger(m, sids) for m in range(core.num_models)])
        if core.pool_models:
            snap['stream_pool'] = core.stream_pool(sids)
            snap['stream_pool_trigger'] = core.stream_pool_trigger(sids)
        return snap

    def import_streams(self, snapshot, ids=None):
        """Continue the snapshot's streams (export_streams of a batch with the same front end and bank) as streams ids (host
        int32 array; None: 0..n-1) of this batch.  Their masks, then each slot's trigger settings, then their pool models,
        then their pool trigger settings are set where they differ from this batch's, so a batch never becomes routed or
        trigger-flagged for nothing; then the state is imported, which overwrites the activations those steps may have
        re-armed.  A snapshot that does not match (pool models this batch does not hold, or pool trigger settings it cannot
        take, included) raises ValueError before anything changes.  History on / off is not
        carried: the streams keep this batch's setting, and one that has history starts empty at the imported sample count."""
        core = self.core
        torch = core.torch
        state = snapshot['state'].to(core.device)
        masks = np.asarray(snapshot['stream_models'], np.uint8)
        trig = snapshot['stream_trigger']
        n = state.shape[0] if state.dim() == 2 else -1
        core._check_state('state', state, n)
        sids = self._host_ids(ids, n)
        _check_np('stream_models', masks, np.uint8, (n,), optional=False)
        if len(trig) != core.num_models:
            raise ValueError('snapshot has trigger settings of %d bank models, this batch has %d' % (len(trig), core.num_models))
        # the record headers against this batch's own, so that the steps below never run for a snapshot import would refuse
        ref = core.export_streams(n=1)[0, :48]
        bad = (state[:, :48] != ref).any(1) | (state[:, 48:56].contiguous().view(torch.int64)[:, 0] < 0)
        pool = None
        if 'stream_pool' in snapshot:        # pool models this batch can take, before anything changes
            pool = np.asarray(snapshot['stream_pool'], np.int32)
            _check_np('stream_pool', pool, np.int32, (n,), optional=False)
            on = pool[pool != -1]
            if on.size and (on.min() < 0 or on.max() >= core.pool_models or not core.pool_loaded[on].all()):
                raise ValueError('snapshot names pool models this batch does not hold (pool of %d slots); nothing was changed'
                                 % core.pool_models)
        ptrig = None
        if 'stream_pool_trigger' in snapshot:    # pool trigger settings this batch can take, before anything changes
            ptrig = snapshot['stream_pool_trigger']
            if not isinstance(ptrig, (tuple, list)) or len(ptrig) != 3:
                raise ValueError('stream_pool_trigger must be (sensitivity, trigger_level, chunk_size); nothing was changed')
            ptrig = [np.asarray(v) for v in ptrig]
            for name, v, kinds in zip(('sensitivity', 'trigger_level', 'chunk_size'), ptrig, ('biuf', 'iu', 'iu')):
                if v.shape != (n,) or v.dtype.kind not in kinds:
                    raise ValueError('stream_pool_trigger %s must be a [%d] array of %s, got %s %s; nothing was changed'
                                     % (name, n, 'real numbers' if kinds == 'biuf' else 'integers', v.dtype, v.shape))
                if kinds == 'iu' and v.size and (int(v.min()) < -2 ** 31 or int(v.max()) >= 2 ** 31):
                    raise ValueError('stream_pool_trigger %s must fit in int32; nothing was changed' % name)
            ptrig = [np.ascontiguousarray(ptrig[0], np.float64), np.ascontiguousarray(ptrig[1], np.int32),
                     np.ascontiguousarray(ptrig[2], np.int32)]
            if n and int(ptrig[2].min()) < 0:
                raise ValueError('stream_pool_trigger chunk_size must be >= 0; nothing was changed')
            if not core.pool_models and ptrig[2].any():
                raise ValueError('snapshot sets pool trigger settings and this batch has no model pool; nothing was changed')
        if n and bool(bad.any()):
            i = int(bad.nonzero()[0, 0])
            got, want = state[i, :48].cpu().numpy().view(np.int32), ref.cpu().numpy().view(np.int32)
            k = np.nonzero(got != want)[0]
            what = ('%s = %d, this batch has %d' % (STATE_FIELDS[k[0]], got[k[0]], want[k[0]])) if k.size else 'n_samples < 0'
            raise ValueError('snapshot record %d does not match this batch: %s; nothing was changed' % (i, what))
        differ = core.stream_models(sids) != masks
        if differ.any():
            core.set_stream_models(masks[differ], sids[differ])
        for slot, (sens, lvl, chunk) in enumerate(trig):
            sens, lvl, chunk = np.asarray(sens, np.float64), np.asarray(lvl, np.int32), np.asarray(chunk, np.int32)
            cs, cl, cc = core.stream_trigger(slot, sids)
            differ = (cs.view(np.uint64) != sens.view(np.uint64)) | (cl != lvl) | (cc != chunk)
            if differ.any():
                core.set_stream_trigger(slot, sens[differ], lvl[differ], chunk[differ], ids=sids[differ])
        if pool is not None:
            differ = core.stream_pool(sids) != pool
            if differ.any():
                core.set_stream_pool(pool[differ], sids[differ])
        if ptrig is not None and core.pool_models:
            sens, lvl, chunk = ptrig
            cs, cl, cc = core.stream_pool_trigger(sids)
            # (NaN, 0, 0) entries follow the model: they differ only from a stream that has its own settings
            differ = (cc != chunk) | ((chunk != 0) & ((cs.view(np.uint64) != sens.view(np.uint64)) | (cl != lvl)))
            if differ.any():
                core.set_stream_pool_trigger(sens[differ], lvl[differ], chunk[differ], ids=sids[differ])
        core.import_streams(state, sids)

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
        self.pool_count.zero_()

    def clear(self, ids=None):
        self.core.clear(ids=ids) if ids is not None else self.core.clear()
