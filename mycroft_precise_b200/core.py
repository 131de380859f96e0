"""ctypes binding of libprecise_b200.so (C ABI: include/precise_b200.h) + a tensor-level wrapper.

PyTorch is used for device memory, streams and (in dist.py) torch.distributed only; every
computation below is a call into the CUDA library.  No fallback: a missing library or device raises.
"""
import ctypes as C
import os

import numpy as np

from .params import ListenerParams

_HERE = os.path.dirname(os.path.abspath(__file__))
PB_MAX_THRESHOLDS = 8
PB_MAX_MODELS = 8
PB_ABI_VERSION = 2
CORPUS_SCHEDULES = {'listener': 0, 'simulate': 1}   # PB_CORPUS_LISTENER, PB_CORPUS_SIMULATE
# ListenerParams fields of the MFCC front end: the models of one handle's bank must agree on all of them
FRONT_END_FIELDS = ('sample_rate', 'window_samples', 'hop_samples', 'n_fft', 'n_filt', 'n_mfcc', 'n_features',
                    'use_delta', 'vectorizer')


class PBError(RuntimeError):
    pass


class pb_config(C.Structure):
    _fields_ = [
        ('abi_version', C.c_int32), ('device', C.c_int32), ('max_streams', C.c_int32),
        ('chunk_samples', C.c_int32),
        ('sample_rate', C.c_int32), ('window_samples', C.c_int32), ('hop_samples', C.c_int32),
        ('n_fft', C.c_int32), ('n_filt', C.c_int32), ('n_mfcc', C.c_int32), ('n_features', C.c_int32),
        ('use_delta', C.c_int32), ('vectorizer', C.c_int32),
        ('hidden', C.c_int32), ('activation', C.c_int32), ('recurrent_activation', C.c_int32),
        ('n_thresholds', C.c_int32),
        ('threshold_mu', C.c_double * PB_MAX_THRESHOLDS), ('threshold_std', C.c_double * PB_MAX_THRESHOLDS),
        ('threshold_center', C.c_double),
        ('sensitivity', C.c_double), ('trigger_level', C.c_int32), ('decode_legacy_f64', C.c_int32),
    ]


PB_TRAIN_STRIDE = 2980             # floats per network of pb_train's weight and accumulator rows
PB_TRAIN_WIDE_STRIDE = 55812       # the same for pb_train_wide (up to 128 GRU units)


class pb_train_row(C.Structure):
    _fields_ = [('hidden', C.c_int32), ('activation', C.c_int32), ('recurrent_activation', C.c_int32), ('seed', C.c_uint32)]


# pb_generate's host tables (pb_gen_item, pb_gen_segment) as numpy records
GEN_ITEM = np.dtype([('background', '<i4'), ('reserved', '<i4'), ('gain', '<f8'), ('length', '<i8'), ('seg_begin', '<i8'),
                     ('seg_end', '<i8')])
GEN_SEGMENT = np.dtype([('clip', '<i4'), ('reserved', '<i4'), ('start', '<i8'), ('length', '<i8')])


class pb_train_opts(C.Structure):
    _fields_ = [('epochs', C.c_int32), ('epoch0', C.c_int32), ('batch_size', C.c_int32), ('lr', C.c_float), ('rho', C.c_float),
                ('epsilon', C.c_float), ('loss_bias', C.c_float), ('dropout', C.c_float)]


# name -> (restype, argtypes); must list every symbol include/precise_b200.h declares
_VP, _I64, _I32 = C.c_void_p, C.c_int64, C.c_int32
SYMBOLS = {
    'pb_config_default': (C.c_int, [C.POINTER(pb_config)]),
    'pb_create': (C.c_int, [C.POINTER(pb_config), C.POINTER(_VP)]),
    'pb_destroy': (None, [_VP]),
    'pb_load_weights': (C.c_int, [_VP, _VP, _VP, _VP, _VP, C.c_float]),
    'pb_mfcc_frames': (_I64, [_VP, _I64]),
    'pb_feature_size': (_I32, [_VP]),
    'pb_mfcc_width': (_I32, [_VP]),
    'pb_mfcc': (C.c_int, [_VP, _VP, _I64, _I64, _VP, _VP]),
    'pb_mfcc_f32': (C.c_int, [_VP, _VP, _I64, _I64, _VP, _VP]),
    'pb_predict': (C.c_int, [_VP, _VP, _I64, _VP, _VP, _VP]),
    'pb_decode': (C.c_int, [_VP, _VP, _I64, _VP, _VP]),
    'pb_update': (C.c_int, [_VP, _VP, _VP, _I64, _VP, _VP, _VP, _VP, _VP]),
    'pb_add_model': (C.c_int, [_VP, C.POINTER(pb_config), _VP, _VP, _VP, _VP, C.c_float, _VP, _I64, C.POINTER(_I32)]),
    'pb_num_models': (C.c_int, [_VP]),
    'pb_update_models': (C.c_int, [_VP, _VP, _VP, _I64, _VP, _VP, _VP, _VP, _VP]),
    'pb_update_ragged': (C.c_int, [_VP, _VP, _VP, _I64, _VP, _I64, _VP, _VP, _VP, _VP, _VP]),
    'pb_update_vectors': (C.c_int, [_VP, _VP, _VP, _I64, _VP]),
    'pb_update_host': (C.c_int, [_VP, _VP, _VP, _I64, _VP, _VP, _VP, _VP]),
    'pb_read_window': (C.c_int, [_VP, _VP, _I64, _VP, _VP]),
    'pb_clear': (C.c_int, [_VP, _VP, _I64, _VP]),
    'pb_set_stream_models': (C.c_int, [_VP, _VP, _VP, _I64]),
    'pb_get_stream_models': (C.c_int, [_VP, _VP, _I64, _VP]),
    'pb_set_stream_trigger': (C.c_int, [_VP, _I32, _VP, _VP, _VP, _VP, _I64]),
    'pb_get_stream_trigger': (C.c_int, [_VP, _I32, _VP, _I64, _VP, _VP, _VP]),
    'pb_stream_state_bytes': (_I64, [_VP]),
    'pb_export_streams': (C.c_int, [_VP, _VP, _I64, _VP, _VP]),
    'pb_import_streams': (C.c_int, [_VP, _VP, _I64, _VP]),
    'pb_set_history': (C.c_int, [_VP, _I64, _I32]),
    'pb_set_stream_history': (C.c_int, [_VP, _VP, _VP, _I64]),
    'pb_get_stream_history': (C.c_int, [_VP, _VP, _I64, _VP]),
    'pb_read_history': (C.c_int, [_VP, _VP, _I64, _I64, _VP, _VP]),
    'pb_set_pool': (C.c_int, [_VP, _I32]),
    'pb_pool_load': (C.c_int, [_VP, _I32, C.POINTER(pb_config), _VP, _VP, _VP, _VP, C.c_float, _VP, _I64]),
    'pb_set_stream_pool': (C.c_int, [_VP, _VP, _VP, _I64]),
    'pb_get_stream_pool': (C.c_int, [_VP, _VP, _I64, _VP]),
    'pb_update_pool': (C.c_int, [_VP, _VP, _VP, _I64, _VP, _I64, _VP, _VP, _VP, _VP, _VP]),
    'pb_update_all': (C.c_int, [_VP, _VP, _VP, _I64, _VP, _I64, _VP, _VP, _VP, _VP, _VP, _VP]),
    'pb_set_stream_pool_trigger': (C.c_int, [_VP, _VP, _VP, _VP, _VP, _I64]),
    'pb_get_stream_pool_trigger': (C.c_int, [_VP, _VP, _I64, _VP, _VP, _VP]),
    'pb_corpus_windows': (_I64, [C.POINTER(pb_config), _I32, _I64, _I64]),
    'pb_score_corpus': (C.c_int, [_VP, _VP, _VP, _I64, _I32, _I32, _I64, C.c_double, _VP, _VP, _VP, _VP, _VP, _VP, _VP]),
    'pb_score_corpus_pool': (C.c_int, [_VP, _VP, _VP, _I64, _VP, _I64, _I32, _I32, _I64, C.c_double, _VP, _VP, _VP, _VP, _VP,
                                       _VP, _VP]),
    'pb_score_corpus_pairs': (C.c_int, [_VP, _VP, _VP, _I64, _VP, _VP, _I64, _I32, _I32, _I64, C.c_double, _VP, _VP, _VP, _VP,
                                        _VP, _VP, C.c_double, _VP, _I64, _VP, _VP]),
    'pb_score_dataset': (C.c_int, [_VP, _VP, _VP, _I64, _VP, _VP, _I64, _VP, _VP, _I64, _I32, _I64, _VP, _I32, _VP, _VP, _VP, _VP,
                                   C.c_double, _VP, _I64, _VP, _VP]),
    'pb_vectorize_clips': (C.c_int, [_VP, _VP, _VP, _I64, _I32, _I64, _VP, _VP]),
    'pb_add_noise': (C.c_int, [_VP, _VP, _VP, _I64, _VP, _I64, _VP, _VP, _I64, _I64, _I32, _I64, _VP, _VP, _VP]),
    'pb_generate': (C.c_int, [_VP, _VP, _VP, _I64, _VP, _VP, _I64, _VP, _I64, _VP, _I64, _VP, _I64, _I64, _I32, _VP, _VP, _VP]),
    'pb_train_opts_default': (C.c_int, [C.POINTER(pb_train_opts)]),
    'pb_train': (C.c_int, [_VP, _VP, _I64, _VP, _VP, _I64, _VP, _VP, _I64, C.POINTER(pb_train_opts), _VP, _VP, _VP, _VP]),
    'pb_train_loss': (C.c_int, [_VP, _VP, _I64, _VP, _VP, _I64, _VP, _VP, _I64, C.c_float, C.c_float, _I32, _VP, _VP, _VP, _VP]),
    'pb_train_wide': (C.c_int, [_VP, _VP, _I64, _VP, _VP, _I64, _VP, _VP, _I64, C.POINTER(pb_train_opts), _VP, _VP, _VP, _VP]),
    'pb_train_wide_loss': (C.c_int, [_VP, _VP, _I64, _VP, _VP, _I64, _VP, _VP, _I64, C.c_float, C.c_float, _I32, _VP, _VP, _VP,
                                     _VP]),
    'pb_score_rows': (C.c_int, [_VP, _VP, _I64, _VP, _VP, _I64, _VP, _I32, _VP, _VP, _I64, _VP, _I32, _VP, _VP, _VP, _VP,
                                C.c_double, _VP, _I64, _VP, _VP]),
    'pb_host_alloc': (C.c_int, [C.POINTER(_VP), C.c_uint64]),
    'pb_host_free': (C.c_int, [_VP]),
    'pb_profile_enable': (C.c_int, [_VP, C.c_int]),
    'pb_profile_reset': (C.c_int, [_VP]),
    'pb_profile_read': (C.c_int, [_VP, C.POINTER(C.c_double), C.POINTER(C.c_uint64)]),
    'pb_get_filterbank': (C.c_int, [_VP, _VP]),
    'pb_get_cdf': (_I64, [_VP, _VP, _I64, C.POINTER(_I32), C.POINTER(_I32)]),
    'pb_set_cdf': (C.c_int, [_VP, _VP, _I64]),
    'pb_debug_force_generic': (C.c_int, [_VP, C.c_int]),
    'pb_debug_gru_mode': (C.c_int, [_VP, C.c_int]),
    'pb_debug_k1_mode': (C.c_int, [_VP, C.c_int]),
    'pb_debug_pool_tiles': (C.c_int, [_VP, C.c_int]),
    'pb_debug_corpus_pool_rows': (C.c_int, [_VP, _I64]),
    'pb_debug_corpus_pool_scan': (C.c_int, [_VP, _I32, _I32]),
    'pb_debug_corpus_pairs_batch': (C.c_int, [_VP, _I64]),
    'pb_debug_rows_groups': (C.c_int, [_VP, _I32, _I64]),
    'pb_debug_tc_dft_power': (C.c_int, [_VP, _VP]),
    'pb_debug_mma_dft_power': (C.c_int, [_VP, _VP]),
    'pb_debug_tc_mfcc_frame': (C.c_int, [_VP, _VP, _VP]),
    'pb_debug_tc3_mfcc_frame': (C.c_int, [_VP, _VP, _VP, _VP]),
    'pb_last_error': (C.c_char_p, []),
    'pb_abi_version': (C.c_int, []),
    'pb_build_info': (C.c_char_p, []),
}

_lib = None


def lib_path() -> str:
    return os.environ.get('PRECISE_B200_LIB', os.path.join(_HERE, 'csrc', 'libprecise_b200.so'))


def get_lib():
    """Load the CUDA library (once).  Fails loudly: there is no other implementation."""
    global _lib
    if _lib is None:
        path = lib_path()
        if not os.path.isfile(path):
            raise PBError('%s is missing: build it with `make -C %s` (or __graft_entry__.build()); '
                          'there is no CPU fallback' % (path, os.path.join(_HERE, 'csrc')))
        lib = C.CDLL(path)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(lib, name)          # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
        if lib.pb_abi_version() != PB_ABI_VERSION:
            raise PBError('ABI mismatch: library %d, binding %d' % (lib.pb_abi_version(), PB_ABI_VERSION))
        _lib = lib
    return _lib


_EXC = {-1: ValueError, -2: NotImplementedError, -3: PBError, -4: PBError, -5: EOFError}


def check(rc: int):
    if rc != 0:
        msg = get_lib().pb_last_error().decode('utf-8', 'replace')
        raise _EXC.get(rc, PBError)(msg)


def make_config(pr: ListenerParams, hidden=20, max_streams=1, chunk_samples=1024, device=0,
                sensitivity=0.5, trigger_level=3, activation='linear',
                recurrent_activation='hard_sigmoid', decode_legacy_f64=False) -> pb_config:
    cfg = pb_config()
    check(get_lib().pb_config_default(C.byref(cfg)))
    cfg.device = device
    cfg.max_streams = max_streams
    cfg.chunk_samples = chunk_samples
    cfg.sample_rate = pr.sample_rate
    cfg.window_samples = pr.window_samples
    cfg.hop_samples = pr.hop_samples
    cfg.n_fft = pr.n_fft
    cfg.n_filt = pr.n_filt
    cfg.n_mfcc = pr.n_mfcc
    cfg.n_features = pr.n_features
    cfg.use_delta = int(pr.use_delta)
    cfg.vectorizer = pr.vectorizer
    cfg.hidden = hidden
    cfg.activation = {'linear': 0, 'tanh': 1}[activation]
    cfg.recurrent_activation = {'hard_sigmoid': 0, 'sigmoid': 1}[recurrent_activation]
    tc = pr.threshold_config
    if not 1 <= len(tc) <= PB_MAX_THRESHOLDS:
        raise ValueError('threshold_config must hold 1..%d (mu, std) pairs' % PB_MAX_THRESHOLDS)
    cfg.n_thresholds = len(tc)
    for i, (mu, std) in enumerate(tc):
        cfg.threshold_mu[i] = mu
        cfg.threshold_std[i] = std
    cfg.threshold_center = pr.threshold_center
    cfg.sensitivity = sensitivity
    cfg.trigger_level = trigger_level
    cfg.decode_legacy_f64 = int(bool(decode_legacy_f64))
    return cfg


def numpy_cdf(threshold_config, resolution=200, min_z=-4, max_z=4):
    """The CDF table exactly as ThresholdDecoder.__init__ builds it (threshold_decoder.py:38-43,
    :68-70, functions.pdf :104-108) -- same numpy calls, so the table is bit-identical to the
    reference's.  This is table construction (6400 doubles, once per handle), not hot-path compute."""
    from math import sqrt, pi
    mu_stds = threshold_config
    min_out = int(min(mu + min_z * std for mu, std in mu_stds))
    max_out = int(max(mu + max_z * std for mu, std in mu_stds))
    out_range = max_out - min_out
    points = np.linspace(min_out, max_out, resolution * out_range)

    def pdf(x, mu, std):
        if std == 0:
            return 0
        return (1.0 / (std * sqrt(2 * pi))) * np.exp(-(x - mu) ** 2 / (2 * std ** 2))

    pd = np.sum([pdf(points, mu, std) for mu, std in mu_stds], axis=0) / (resolution * len(mu_stds))
    return np.ascontiguousarray(np.cumsum(pd), dtype=np.float64), min_out, max_out


def threshold_encode(threshold_config, center, thresholds):
    """ThresholdDecoder.encode (threshold_decoder.py:59-66) of each decoded threshold: the network output it stands for,
    from the same table numpy_cdf builds for the decoder."""
    from math import exp
    cd, min_out, max_out = numpy_cdf(threshold_config)
    out = []
    for t in thresholds:
        t = 0.5 * float(t) / center
        cp = t * center * 2 if t < 0.5 else (t - 0.5) * 2 * (1 - center) + center
        ratio = np.searchsorted(cd, cp) / len(cd)
        out.append(1 / (1 + exp(-(min_out + (max_out - min_out) * ratio))))
    return np.asarray(out, np.float64)


def _schedule(schedule) -> int:
    if schedule in CORPUS_SCHEDULES:
        return CORPUS_SCHEDULES[schedule]
    if isinstance(schedule, (int, np.integer)) and not isinstance(schedule, bool) and int(schedule) in CORPUS_SCHEDULES.values():
        return int(schedule)
    raise ValueError('schedule must be one of %s, got %r' % (sorted(CORPUS_SCHEDULES), schedule))


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _np_ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _check_np(name, a, dtype, shape, optional=True):
    """The C ABI takes raw host pointers: refuse anything whose dtype / shape / layout it would misread."""
    if a is None:
        if optional:
            return
        raise ValueError('%s is required' % name)
    if not isinstance(a, np.ndarray) or a.dtype != np.dtype(dtype) or not a.flags.c_contiguous or tuple(a.shape) != tuple(shape):
        raise ValueError('%s must be a C-contiguous %s array of shape %s, got %s %s' % (
            name, np.dtype(dtype).name, tuple(shape), getattr(a, 'dtype', type(a)), getattr(a, 'shape', None)))


class PreciseB200:
    """One library handle: tables + per-stream state for ``max_streams`` streams on one GPU.

    Tensor-level API (torch CUDA tensors in, torch CUDA tensors out, asynchronous on the current
    torch stream).  Higher-level mirrors of the reference classes live in runner.py / batch.py.
    """

    def __init__(self, params: ListenerParams = None, hidden=20, max_streams=1, chunk_samples=1024,
                 device=0, sensitivity=0.5, trigger_level=3, activation='linear',
                 recurrent_activation='hard_sigmoid', decode_legacy_f64=False, check_ids=False):
        import torch
        self.torch = torch
        self.lib = get_lib()
        self.params = params or ListenerParams()
        if not torch.cuda.is_available():
            raise PBError('no CUDA device: mycroft_precise_b200 has no CPU path')
        self.device = torch.device('cuda', device)
        self.cfg = make_config(self.params, hidden, max_streams, chunk_samples, device, sensitivity,
                               trigger_level, activation, recurrent_activation, decode_legacy_f64)
        self.check_ids = bool(check_ids)      # debug: also verify 0 <= ids < max_streams and uniqueness (a device sync)
        h = C.c_void_p()
        check(self.lib.pb_create(C.byref(self.cfg), C.byref(h)))
        self._h = h
        self.max_streams = max_streams
        self.chunk_samples = chunk_samples
        self.hidden = hidden
        self.n_features = self.params.n_features
        self.mfcc_width = int(self.lib.pb_mfcc_width(h))
        self.feature_size = int(self.lib.pb_feature_size(h))
        cd, lo, hi = numpy_cdf(self.params.threshold_config)
        if hi > lo:                      # out_range 0 (threshold_decoder.py:48-49): the table is never indexed
            check(self.lib.pb_set_cdf(h, cd.ctypes.data_as(C.c_void_p), len(cd)))
        self._count = torch.zeros(1, dtype=torch.int64, device=self.device)
        self.history_samples = 0             # set_history's samples; 0 = no history pool
        self.pool_models = 0                 # set_pool's max_models; 0 = no model pool
        self.pool_loaded = np.zeros(0, bool)  # which pool slots hold a model
        self._pool_cdfs = {}                 # numpy CDF tables of pool_load, by threshold_config

    def close(self):
        if getattr(self, '_h', None):
            self.lib.pb_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self):
        return C.c_void_p(self.torch.cuda.current_stream(self.device).cuda_stream)

    # ---- model
    @staticmethod
    def _weights(F, H, kernel, recurrent, bias, dense_w):
        k = np.ascontiguousarray(kernel, dtype=np.float32)
        u = np.ascontiguousarray(recurrent, dtype=np.float32)
        b = np.ascontiguousarray(bias, dtype=np.float32).reshape(-1)
        w = np.ascontiguousarray(dense_w, dtype=np.float32).reshape(-1)
        if k.shape != (F, 3 * H) or u.shape != (H, 3 * H) or b.shape != (3 * H,) or w.shape != (H,):
            raise ValueError('weight shapes %s %s %s %s do not match F=%d, H=%d' % (k.shape, u.shape, b.shape, w.shape, F, H))
        return k, u, b, w

    def load_weights(self, kernel, recurrent, bias, dense_w, dense_b):
        k, u, b, w = self._weights(self.feature_size, self.hidden, kernel, recurrent, bias, dense_w)
        vp = lambda a: a.ctypes.data_as(C.c_void_p)
        check(self.lib.pb_load_weights(self._h, vp(k), vp(u), vp(b), vp(w), float(np.asarray(dense_b).reshape(-1)[0])))

    # ---- model bank: more networks over the same MFCC front end (slot 0 is the network of load_weights)
    def _model_args(self, model, params, sensitivity, trigger_level, decode_legacy_f64, cdf):
        """(cfg, weights, CDF table or None) of a network for this handle's front end, as add_model and pool_load take it."""
        from .runner import _resolve_model
        model, pr = _resolve_model(model)
        pr = params or pr or self.params
        diff = [f for f in FRONT_END_FIELDS if getattr(pr, f) != getattr(self.params, f)]
        if diff:
            raise ValueError('front end of the model differs from the handle in %s: the models of a bank share one MFCC front end'
                             % ', '.join('%s (%r != %r)' % (f, getattr(pr, f), getattr(self.params, f)) for f in diff))
        if model.feature_size != self.feature_size:
            raise ValueError('model expects %d features, the handle computes %d' % (model.feature_size, self.feature_size))
        cfg = make_config(pr, model.hidden, self.max_streams, self.chunk_samples, self.device.index, sensitivity,
                          trigger_level, model.activation, model.recurrent_activation, decode_legacy_f64)
        k, u, b, w = self._weights(self.feature_size, model.hidden, model.kernel, model.recurrent, model.bias, model.dense_w)
        cd, lo, hi = cdf(pr.threshold_config)
        return cfg, (k, u, b, w, float(model.dense_b)), (cd if hi > lo else None)

    def add_model(self, model, params: ListenerParams = None, sensitivity=0.5, trigger_level=3, decode_legacy_f64=False) -> int:
        """Add a network to this handle's bank; returns its slot.  ``model`` is a GruModel or a .npz / .pb / .net path (its
        .params file is read as the reference does).  ``params`` (else the model's .params, else this handle's params) gives
        the model's decoder settings; its front end must equal this handle's."""
        cfg, (k, u, b, w, bd), cd = self._model_args(model, params, sensitivity, trigger_level, decode_legacy_f64, numpy_cdf)
        vp = lambda a: a.ctypes.data_as(C.c_void_p)
        slot = C.c_int32(-1)
        check(self.lib.pb_add_model(self._h, C.byref(cfg), vp(k), vp(u), vp(b), vp(w), bd, _np_ptr(cd),
                                    0 if cd is None else len(cd), C.byref(slot)))
        return int(slot.value)

    # ---- model pool: up to 2^24 networks of the fused family, at most one per stream (pb_set_pool in precise_b200.h)
    def set_pool(self, max_models):
        """A model pool of ``max_models`` empty slots, every stream on none.  Calling it again replaces the pool and
        unassigns every stream; 0 frees it.  Synchronous."""
        max_models = self._int('max_models', max_models)
        if not -2 ** 31 <= max_models < 2 ** 31:
            raise ValueError('max_models must fit in int32, got %d' % max_models)
        rc = self.lib.pb_set_pool(self._h, max_models)
        if rc != -1:                         # anything but a refused argument replaced the pool
            self.pool_models = max_models if rc == 0 else 0
            self.pool_loaded = np.zeros(self.pool_models, bool)
        check(rc)

    def _pool_cdf(self, threshold_config):
        key = tuple(tuple(float(x) for x in p) for p in threshold_config)
        if key not in self._pool_cdfs:
            self._pool_cdfs[key] = numpy_cdf(threshold_config)
        return self._pool_cdfs[key]

    def pool_load(self, model_id, model, params: ListenerParams = None, sensitivity=0.5, trigger_level=3,
                  decode_legacy_f64=False):
        """Load a network (GruModel or weights path, as add_model takes it) into pool slot ``model_id``, replacing what the
        slot held; streams on the slot get fresh detectors.  Networks outside the fused family (hidden <= 24, no deltas) raise
        NotImplementedError.  Synchronous."""
        model_id = self._slot(model_id)
        cfg, (k, u, b, w, bd), cd = self._model_args(model, params, sensitivity, trigger_level, decode_legacy_f64, self._pool_cdf)
        vp = lambda a: a.ctypes.data_as(C.c_void_p)
        check(self.lib.pb_pool_load(self._h, model_id, C.byref(cfg), vp(k), vp(u), vp(b), vp(w), bd, _np_ptr(cd),
                                    0 if cd is None else len(cd)))
        self.pool_loaded[model_id] = True

    def set_stream_pool(self, model_ids, ids=None):
        """Stream ids[i] (host int32 array; None: stream i) goes to pool slot model_ids[i] (host int32 array, -1 = none).  A
        stream whose model changes gets a fresh detector.  Synchronous; bad input raises ValueError and changes nothing."""
        model_ids = np.asarray(model_ids)
        n = model_ids.shape[0] if model_ids.ndim == 1 else -1
        _check_np('model_ids', model_ids, np.int32, (n,), optional=False)
        _check_np('ids', ids, np.int32, (n,))
        check(self.lib.pb_set_stream_pool(self._h, _np_ptr(ids), _np_ptr(model_ids), n))

    def stream_pool(self, ids=None) -> np.ndarray:
        """int32 pool model of streams ids (host int32 array), or of every stream; -1 = none."""
        n = self.max_streams if ids is None else (ids.shape[0] if isinstance(ids, np.ndarray) and ids.ndim == 1 else -1)
        _check_np('ids', ids, np.int32, (n,))
        out = np.zeros(n, np.int32)
        check(self.lib.pb_get_stream_pool(self._h, _np_ptr(ids), n, _np_ptr(out)))
        return out

    def update_pool(self, pcm, ids=None, offsets=None, max_len=None, out=None, count=None):
        """Pool tick: each item scored by its stream's pool model.  Without ``offsets``, pcm is int16 CUDA [n, chunk_samples]
        (update's tick); with them, a 1-D int16 CUDA pcm and int64 CUDA offsets [n + 1] (update_ragged's tick).  Returns
        dict(raw f32, conf f64, fired u8), each [n]; items whose stream has no pool model are NaN / NaN / 0.  ``count``
        (int64 [1]) accumulates the tick's pool fires."""
        n, max_len = self._tick_shape(pcm, offsets, max_len)
        self._check_ids(ids, n)
        out = self._tick_out(out, 1, n, (n,))
        self._check_t('count', count, self.torch.int64, 1)
        check(self.lib.pb_update_pool(self._h, _ptr(pcm), _ptr(offsets), max_len, _ptr(ids), n, _ptr(out.get('raw')),
                                      _ptr(out['conf']), _ptr(out.get('fired')), _ptr(count), self._stream()))
        return out

    def update_all(self, pcm, ids=None, offsets=None, max_len=None, out=None, counts=None, pool_count=None):
        """Combined tick: the bank and the pool on one chunk, with one history append and one K1.  pcm and ``offsets`` as
        update_pool takes them (uniform without offsets, ragged with them).  Returns dict(raw f32, conf f64, fired u8), each
        [M + 1, n]: rows 0 .. M-1 are update_models's (update_ragged's with offsets), row M is update_pool's.  ``counts``
        (int64 [M]) accumulates each bank model's fires and ``pool_count`` (int64 [1]) the pool's."""
        n, max_len = self._tick_shape(pcm, offsets, max_len)
        self._check_ids(ids, n)
        M = self.num_models
        out = self._tick_out(out, M + 1, n, (M + 1, n))
        self._check_t('counts', counts, self.torch.int64, M)
        self._check_t('pool_count', pool_count, self.torch.int64, 1)
        check(self.lib.pb_update_all(self._h, _ptr(pcm), _ptr(offsets), max_len, _ptr(ids), n, _ptr(out.get('raw')),
                                     _ptr(out['conf']), _ptr(out.get('fired')), _ptr(counts), _ptr(pool_count),
                                     self._stream()))
        return out

    def _tick_shape(self, pcm, offsets, max_len):
        """(n, max_len) of a tick that is uniform without ``offsets`` and ragged with them, as update_pool takes it."""
        torch = self.torch
        if offsets is None:
            return self._check_pcm(pcm), 0
        if (not isinstance(pcm, torch.Tensor) or pcm.dtype != torch.int16 or pcm.dim() != 1 or not pcm.is_contiguous()
                or pcm.device != self.device):
            raise ValueError('pcm must be a contiguous 1-D int16 tensor on %s' % self.device)
        if (not isinstance(offsets, torch.Tensor) or offsets.dtype != torch.int64 or offsets.dim() != 1 or offsets.numel() < 1
                or not offsets.is_contiguous() or offsets.device != self.device):
            raise ValueError('offsets must be a contiguous 1-D int64 [n + 1] tensor on %s' % self.device)
        n = offsets.numel() - 1
        if n > self.max_streams:
            raise ValueError('n = %d exceeds max_streams = %d' % (n, self.max_streams))
        if max_len is None:
            max_len = max(1, int((offsets[1:] - offsets[:-1]).max())) if n else 1
        max_len = int(max_len)
        if max_len < 1:
            raise ValueError('max_len must be >= 1, got %d' % max_len)
        return n, max_len

    def _tick_out(self, out, rows, n, shape):
        """``out`` checked for ``rows`` x n outputs, or new buffers of ``shape``."""
        torch = self.torch
        if out is not None:
            self._check_t("out['raw']", out.get('raw'), torch.float32, rows * n)
            self._check_t("out['conf']", out.get('conf'), torch.float64, rows * n, optional=False)
            self._check_t("out['fired']", out.get('fired'), torch.uint8, rows * n)
            return out
        return dict(raw=torch.empty(shape, dtype=torch.float32, device=self.device),
                    conf=torch.empty(shape, dtype=torch.float64, device=self.device),
                    fired=torch.empty(shape, dtype=torch.uint8, device=self.device))

    def set_stream_pool_trigger(self, sensitivity, trigger_level, chunk_size, ids=None):
        """Stream ids[i] is scored by TriggerDetector(chunk_size[i], sensitivity[i], trigger_level[i]) on whichever pool model
        it is on.  ``chunk_size`` is in BYTES; 0 returns the stream to its model's own settings.  Scalars broadcast as in
        set_stream_trigger.  A stream whose entry changes gets a fresh pool detector; an unchanged entry keeps it.  The
        settings survive set_stream_pool, pool_load and clear; set_pool drops them.  Synchronous; bad input raises ValueError
        and changes nothing."""
        ids, sens, level, chunk, n = self._trigger_args(sensitivity, trigger_level, chunk_size, ids, 0)
        check(self.lib.pb_set_stream_pool_trigger(self._h, _np_ptr(ids), _np_ptr(sens), _np_ptr(level), _np_ptr(chunk), n))

    def stream_pool_trigger(self, ids=None):
        """(sensitivity f64[n], trigger_level i32[n], chunk_size i32[n], in bytes) of the pool settings of streams ids (host
        int32 array), or of every stream.  A stream that follows its model reports (NaN, 0, 0)."""
        n = self.max_streams if ids is None else (ids.shape[0] if isinstance(ids, np.ndarray) and ids.ndim == 1 else -1)
        _check_np('ids', ids, np.int32, (n,))
        sens, level, chunk = np.zeros(n, np.float64), np.zeros(n, np.int32), np.zeros(n, np.int32)
        check(self.lib.pb_get_stream_pool_trigger(self._h, _np_ptr(ids), n, _np_ptr(sens), _np_ptr(level), _np_ptr(chunk)))
        return sens, level, chunk

    @property
    def num_models(self) -> int:
        return int(self.lib.pb_num_models(self._h))

    # ---- stateless pieces
    def mfcc_frames(self, n_samples: int) -> int:
        return int(self.lib.pb_mfcc_frames(self._h, n_samples))

    def mfcc(self, pcm):
        """pcm [S, L] int16 or float32 CUDA tensor -> [S, n_frames, mfcc_width] float32."""
        torch = self.torch
        if pcm.dim() == 1:
            pcm = pcm[None]
        pcm = pcm.contiguous()
        S, L = pcm.shape
        nf = self.mfcc_frames(L)
        out = torch.empty((S, nf, self.mfcc_width), dtype=torch.float32, device=self.device)
        if pcm.dtype == torch.int16:
            check(self.lib.pb_mfcc(self._h, _ptr(pcm), S, L, _ptr(out), self._stream()))
        elif pcm.dtype == torch.float32:
            check(self.lib.pb_mfcc_f32(self._h, _ptr(pcm), S, L, _ptr(out), self._stream()))
        else:
            raise ValueError('pcm must be int16 or float32')
        return out

    def predict(self, inputs, want_logit=False):
        """inputs [N, n_features, feature_size] float32 CUDA -> prob [N] float32 (Runner.predict)."""
        torch = self.torch
        inputs = inputs.contiguous()
        if inputs.dim() != 3 or inputs.shape[1] != self.n_features or inputs.shape[2] != self.feature_size:
            raise ValueError('inputs must be [N, %d, %d], got %s' % (self.n_features, self.feature_size, tuple(inputs.shape)))
        if inputs.dtype != torch.float32:
            raise ValueError('inputs must be float32')
        N = inputs.shape[0]
        out = torch.empty(N, dtype=torch.float32, device=self.device)
        logit = torch.empty(N, dtype=torch.float32, device=self.device) if want_logit else None
        check(self.lib.pb_predict(self._h, _ptr(inputs), N, _ptr(out), _ptr(logit), self._stream()))
        return (out, logit) if want_logit else out

    def decode(self, raw):
        torch = self.torch
        raw = raw.contiguous().to(torch.float32)
        out = torch.empty(raw.numel(), dtype=torch.float64, device=self.device)
        check(self.lib.pb_decode(self._h, _ptr(raw), raw.numel(), _ptr(out), self._stream()))
        return out.view(raw.shape)

    # ---- argument checks: the C ABI reads raw device pointers, so dtype / device / size / layout are verified here
    def _check_t(self, name, t, dtype, numel, optional=True):
        if t is None:
            if optional:
                return
            raise ValueError('%s is required' % name)
        if (not isinstance(t, self.torch.Tensor) or t.dtype != dtype or t.device != self.device
                or t.numel() != numel or not t.is_contiguous()):
            raise ValueError('%s must be a contiguous %s tensor with %d elements on %s, got %s %s on %s' % (
                name, dtype, numel, self.device, getattr(t, 'dtype', type(t)), tuple(getattr(t, 'shape', ())),
                getattr(t, 'device', None)))

    def _check_ids(self, ids, n):
        self._check_t('ids', ids, self.torch.int32, n)
        if ids is not None and self.check_ids and n:
            lo, hi = int(ids.min()), int(ids.max())
            if lo < 0 or hi >= self.max_streams:
                raise ValueError('stream ids must lie in [0, %d), got [%d, %d]' % (self.max_streams, lo, hi))
            if int(self.torch.unique(ids).numel()) != n:
                raise ValueError('stream ids must be unique within a tick')

    def _check_pcm(self, pcm):
        torch = self.torch
        if (not isinstance(pcm, torch.Tensor) or pcm.dtype != torch.int16 or pcm.dim() != 2 or pcm.shape[1] != self.chunk_samples
                or not pcm.is_contiguous() or pcm.device != self.device):
            raise ValueError('pcm must be a contiguous int16 [n, %d] tensor on %s' % (self.chunk_samples, self.device))
        if pcm.shape[0] > self.max_streams:
            raise ValueError('n = %d exceeds max_streams = %d' % (pcm.shape[0], self.max_streams))
        return pcm.shape[0]

    # ---- stateful tick
    def update(self, pcm, ids=None, out=None, count=None):
        """pcm [n, chunk_samples] int16 CUDA.  Returns dict(raw, conf, fired) (+ count accumulates)."""
        torch = self.torch
        n = self._check_pcm(pcm)
        self._check_ids(ids, n)
        if out is not None:
            self._check_t("out['raw']", out.get('raw'), torch.float32, n)
            self._check_t("out['conf']", out.get('conf'), torch.float64, n, optional=False)
            self._check_t("out['fired']", out.get('fired'), torch.uint8, n)
        self._check_t('count', count, torch.int64, 1)
        if out is None:
            out = dict(raw=torch.empty(n, dtype=torch.float32, device=self.device),
                       conf=torch.empty(n, dtype=torch.float64, device=self.device),
                       fired=torch.empty(n, dtype=torch.uint8, device=self.device))
        check(self.lib.pb_update(self._h, _ptr(pcm), _ptr(ids), n, _ptr(out.get('raw')), _ptr(out['conf']),
                                 _ptr(out.get('fired')), _ptr(count), self._stream()))
        return out

    def update_models(self, pcm, ids=None, out=None, counts=None):
        """Bank tick: pcm [n, chunk_samples] int16 CUDA.  Returns dict(raw f32, conf f64, fired u8), each [M, n] for the M
        models of the bank (slot order); ``counts`` (int64 [M]) accumulates each model's fired streams."""
        torch = self.torch
        n = self._check_pcm(pcm)
        self._check_ids(ids, n)
        M = self.num_models
        if out is not None:
            self._check_t("out['raw']", out.get('raw'), torch.float32, M * n)
            self._check_t("out['conf']", out.get('conf'), torch.float64, M * n, optional=False)
            self._check_t("out['fired']", out.get('fired'), torch.uint8, M * n)
        self._check_t('counts', counts, torch.int64, M)
        if out is None:
            out = dict(raw=torch.empty((M, n), dtype=torch.float32, device=self.device),
                       conf=torch.empty((M, n), dtype=torch.float64, device=self.device),
                       fired=torch.empty((M, n), dtype=torch.uint8, device=self.device))
        check(self.lib.pb_update_models(self._h, _ptr(pcm), _ptr(ids), n, _ptr(out.get('raw')), _ptr(out['conf']),
                                        _ptr(out.get('fired')), _ptr(counts), self._stream()))
        return out

    def update_ragged(self, pcm, offsets, ids=None, max_len=None, out=None, counts=None):
        """Ragged bank tick: stream item i brings pcm[offsets[i]:offsets[i + 1]] (any length >= 1, any alignment) this tick.
        pcm is a 1-D int16 CUDA tensor, offsets an int64 CUDA tensor [n + 1].  ``max_len`` bounds every length (None: computed
        here, one device sync).  Returns dict(raw f32, conf f64, fired u8), each [M, n], as update_models; ``counts`` (int64
        [M]) accumulates.  With check_ids, offsets must also be non-decreasing, within pcm, with every length in [1, max_len]."""
        torch = self.torch
        if (not isinstance(pcm, torch.Tensor) or pcm.dtype != torch.int16 or pcm.dim() != 1 or not pcm.is_contiguous()
                or pcm.device != self.device):
            raise ValueError('pcm must be a contiguous 1-D int16 tensor on %s' % self.device)
        if (not isinstance(offsets, torch.Tensor) or offsets.dtype != torch.int64 or offsets.dim() != 1 or offsets.numel() < 1
                or not offsets.is_contiguous() or offsets.device != self.device):
            raise ValueError('offsets must be a contiguous 1-D int64 [n + 1] tensor on %s' % self.device)
        n = offsets.numel() - 1
        if n > self.max_streams:
            raise ValueError('n = %d exceeds max_streams = %d' % (n, self.max_streams))
        self._check_ids(ids, n)
        lens = offsets[1:] - offsets[:-1]
        if max_len is None:
            max_len = max(1, int(lens.max())) if n else 1
        max_len = int(max_len)
        if max_len < 1:
            raise ValueError('max_len must be >= 1, got %d' % max_len)
        if self.check_ids and n:
            lo, hi = int(lens.min()), int(lens.max())
            if lo < 1 or hi > max_len:
                raise ValueError('chunk lengths must lie in [1, max_len = %d], got [%d, %d] (offsets must be non-decreasing)'
                                 % (max_len, lo, hi))
            first, last = int(offsets[0]), int(offsets[-1])
            if first < 0 or last > pcm.numel():
                raise ValueError('offsets [%d, %d] outside pcm of %d samples' % (first, last, pcm.numel()))
        M = self.num_models
        if out is not None:
            self._check_t("out['raw']", out.get('raw'), torch.float32, M * n)
            self._check_t("out['conf']", out.get('conf'), torch.float64, M * n, optional=False)
            self._check_t("out['fired']", out.get('fired'), torch.uint8, M * n)
        self._check_t('counts', counts, torch.int64, M)
        if out is None:
            out = dict(raw=torch.empty((M, n), dtype=torch.float32, device=self.device),
                       conf=torch.empty((M, n), dtype=torch.float64, device=self.device),
                       fired=torch.empty((M, n), dtype=torch.uint8, device=self.device))
        check(self.lib.pb_update_ragged(self._h, _ptr(pcm), _ptr(offsets), max_len, _ptr(ids), n, _ptr(out.get('raw')),
                                        _ptr(out['conf']), _ptr(out.get('fired')), _ptr(counts), self._stream()))
        return out

    def update_vectors(self, pcm, ids=None):
        n = self._check_pcm(pcm)
        self._check_ids(ids, n)
        check(self.lib.pb_update_vectors(self._h, _ptr(pcm), _ptr(ids), n, self._stream()))

    def read_window(self, n=None, ids=None):
        torch = self.torch
        n = (ids.numel() if ids is not None else (self.max_streams if n is None else n))
        self._check_ids(ids, n)
        out = torch.empty((n, self.n_features, self.mfcc_width), dtype=torch.float32, device=self.device)
        check(self.lib.pb_read_window(self._h, _ptr(ids), n, _ptr(out), self._stream()))
        return out

    def clear(self, n=None, ids=None):
        n = (ids.numel() if ids is not None else (self.max_streams if n is None else n))
        self._check_ids(ids, n)
        check(self.lib.pb_clear(self._h, _ptr(ids), n, self._stream()))

    # ---- per-stream model subscriptions
    def set_stream_models(self, masks, ids=None):
        """Bit m of masks[i] = bank slot m scores stream ids[i] (ids None: stream i).  Host numpy arrays: uint8 masks [n],
        int32 ids [n].  Unsubscribed (item, model) pairs of later ticks come back as raw NaN, conf NaN, fired 0, with that
        model's trigger and count untouched; a bit going from 0 to 1 re-arms the model's trigger for the stream.  Streams
        start at 0xFF (every model, including models added later).  Synchronous; bad ids raise ValueError and change nothing."""
        masks = np.asarray(masks)
        n = masks.shape[0] if masks.ndim == 1 else -1
        _check_np('masks', masks, np.uint8, (n,), optional=False)
        _check_np('ids', ids, np.int32, (n,))
        check(self.lib.pb_set_stream_models(self._h, _np_ptr(ids), _np_ptr(masks), n))

    def stream_models(self, ids=None) -> np.ndarray:
        """uint8 masks of streams ids (host int32 array), or of every stream."""
        n = self.max_streams if ids is None else (ids.shape[0] if isinstance(ids, np.ndarray) and ids.ndim == 1 else -1)
        _check_np('ids', ids, np.int32, (n,))
        out = np.zeros(n, np.uint8)
        check(self.lib.pb_get_stream_models(self._h, _np_ptr(ids), n, _np_ptr(out)))
        return out

    # ---- per-stream TriggerDetector settings
    @staticmethod
    def _slot(slot):
        if isinstance(slot, (bool, np.bool_)) or not isinstance(slot, (int, np.integer)) or not -2 ** 31 <= slot < 2 ** 31:
            raise ValueError('slot must be an int32, got %r' % (slot,))
        return int(slot)

    def set_stream_trigger(self, slot, sensitivity, trigger_level, chunk_size, ids=None):
        """Bank slot ``slot`` scores stream ids[i] as TriggerDetector(chunk_size[i], sensitivity[i], trigger_level[i]) would
        (runner.py:121).  ``chunk_size`` is in BYTES, as the reference's TriggerDetector takes it.  Scalars broadcast to the
        ids; ids (host int32 array) None: streams 0..n-1, n = the length of the array arguments, or every stream when all three
        are scalars.  A stream whose values change gets a fresh detector; unchanged values keep its state.  Synchronous; bad
        input raises ValueError and changes nothing."""
        slot = self._slot(slot)
        ids, sens, level, chunk, n = self._trigger_args(sensitivity, trigger_level, chunk_size, ids, 1)
        check(self.lib.pb_set_stream_trigger(self._h, slot, _np_ptr(ids), _np_ptr(sens), _np_ptr(level), _np_ptr(chunk), n))

    def _trigger_args(self, sensitivity, trigger_level, chunk_size, ids, min_chunk):
        """(ids, sensitivity f64[n], trigger_level i32[n], chunk_size i32[n], n) of a trigger setter, scalars broadcast;
        ValueError for anything the C ABI would misread or refuse, chunk sizes below ``min_chunk`` included."""
        vals = [np.asarray(sensitivity), np.asarray(trigger_level), np.asarray(chunk_size)]
        if any(v.ndim > 1 for v in vals):
            raise ValueError('sensitivity, trigger_level and chunk_size must be scalars or 1-D arrays')
        if ids is not None:
            if not isinstance(ids, np.ndarray) or ids.ndim != 1:
                raise ValueError('ids must be a 1-D int32 array')
            n = ids.shape[0]
        else:
            lens = {v.shape[0] for v in vals if v.ndim == 1}
            if len(lens) > 1:
                raise ValueError('sensitivity, trigger_level and chunk_size have different lengths %s' % sorted(lens))
            n = lens.pop() if lens else self.max_streams
        _check_np('ids', ids, np.int32, (n,))
        for name, v in zip(('sensitivity', 'trigger_level', 'chunk_size'), vals):
            if v.ndim == 1 and v.shape[0] != n:
                raise ValueError('%s has %d entries for %d streams' % (name, v.shape[0], n))
        sens, level, chunk = vals
        if sens.dtype.kind not in 'biuf':
            raise ValueError('sensitivity must be real numbers, got %s' % sens.dtype)
        for name, v in (('trigger_level', level), ('chunk_size', chunk)):
            if v.dtype.kind not in 'iu':
                raise ValueError('%s must be integers, got %s' % (name, v.dtype))
            if v.size and (int(v.min()) < -2 ** 31 or int(v.max()) >= 2 ** 31):
                raise ValueError('%s must fit in int32' % name)
        if chunk.size and int(chunk.min()) < min_chunk:
            if min_chunk == 1:
                raise ValueError('chunk_size must be >= 1 byte (TriggerDetector divides by it), got %d' % int(chunk.min()))
            raise ValueError('chunk_size must be >= 0 bytes (0: the model\'s own settings), got %d' % int(chunk.min()))
        sens = np.ascontiguousarray(np.broadcast_to(sens, (n,)), dtype=np.float64)
        level = np.ascontiguousarray(np.broadcast_to(level, (n,)), dtype=np.int32)
        chunk = np.ascontiguousarray(np.broadcast_to(chunk, (n,)), dtype=np.int32)
        return ids, sens, level, chunk, n

    def stream_trigger(self, slot, ids=None):
        """(sensitivity f64[n], trigger_level i32[n], chunk_size i32[n], in bytes) of bank slot ``slot`` for streams ids
        (host int32 array), or for every stream.  Streams never set report the model's own values."""
        slot = self._slot(slot)
        n = self.max_streams if ids is None else (ids.shape[0] if isinstance(ids, np.ndarray) and ids.ndim == 1 else -1)
        _check_np('ids', ids, np.int32, (n,))
        sens, level, chunk = np.zeros(n, np.float64), np.zeros(n, np.int32), np.zeros(n, np.int32)
        check(self.lib.pb_get_stream_trigger(self._h, slot, _np_ptr(ids), n, _np_ptr(sens), _np_ptr(level), _np_ptr(chunk)))
        return sens, level, chunk

    # ---- stream state export / import
    @property
    def stream_state_bytes(self) -> int:
        """Bytes of one stream's state record (layout: include/precise_b200.h); equal on every handle with this front end."""
        b = int(self.lib.pb_stream_state_bytes(self._h))
        if b < 0:
            check(b)
        return b

    def _check_state(self, name, t, n):
        B = self.stream_state_bytes
        if not isinstance(t, self.torch.Tensor) or tuple(t.shape) != (n, B):
            raise ValueError('%s must be a [n, %d] uint8 tensor of stream state records, got shape %s'
                             % (name, B, tuple(getattr(t, 'shape', ()))))
        self._check_t(name, t, self.torch.uint8, n * B, optional=False)

    def export_streams(self, ids=None, n=None, out=None):
        """The state records of streams ids (int32 CUDA tensor; None: streams 0..n-1, n defaulting to max_streams): a uint8
        CUDA tensor [n, stream_state_bytes], written into ``out`` when given.  Asynchronous on the current stream, after the
        ticks queued before it; reads state only."""
        torch = self.torch
        n = ids.numel() if ids is not None else (self.max_streams if n is None else n)
        self._check_ids(ids, n)
        if out is None:
            out = torch.empty((n, self.stream_state_bytes), dtype=torch.uint8, device=self.device)
        else:
            self._check_state('out', out, n)
        check(self.lib.pb_export_streams(self._h, _ptr(ids), n, _ptr(out), self._stream()))
        return out

    def import_streams(self, state, ids=None):
        """Overwrite streams ids[i] (host int32 array, unique; None: streams 0..n-1) with record i of ``state``, a uint8 tensor
        [n, stream_state_bytes] on this handle's device from export_streams of a handle with the same front end and bank
        size (its chunk_samples may differ).  Bank slot m's trigger state goes to slot m.  The streams keep this handle's
        masks and trigger settings.  Synchronous; a bad record or id raises ValueError and changes nothing."""
        n = state.shape[0] if isinstance(state, self.torch.Tensor) and state.dim() == 2 else -1
        self._check_state('state', state, n)
        _check_np('ids', ids, np.int32, (n,))
        check(self.lib.pb_import_streams(self._h, _np_ptr(ids), n, _ptr(state)))

    # ---- stream audio history
    @staticmethod
    def _int(name, v):
        if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)):
            raise ValueError('%s must be an integer, got %r' % (name, v))
        return int(v)

    def set_history(self, samples=None, max_rows=None):
        """A device pool of ``max_rows`` rows (default max_streams), each holding the last ``samples`` int16 samples (default
        params.buffer_samples, the clip the reference's listen.py saves) of one stream that has history.  Every stream starts
        off (set_stream_history switches them on); calling it again replaces the pool, (0, 0) frees it.  Synchronous."""
        samples = self._int('samples', self.params.buffer_samples if samples is None else samples)
        max_rows = self._int('max_rows', self.max_streams if max_rows is None else max_rows)
        if not -2 ** 31 <= max_rows < 2 ** 31:
            raise ValueError('max_rows must fit in int32, got %d' % max_rows)
        rc = self.lib.pb_set_history(self._h, samples, max_rows)
        if rc != -1:                         # anything but a refused argument replaced the pool
            self.history_samples = samples if rc == 0 else 0
        check(rc)

    def set_stream_history(self, on, ids=None):
        """Switch history on (true) or off for streams ids (host int32 array; None: streams 0..n-1, n = len(on), or every
        stream when ``on`` is a scalar, which broadcasts).  A stream that goes on starts empty; one already on keeps its audio.
        Synchronous; bad input, or more streams on than the pool's rows, raises ValueError and changes nothing."""
        on = np.asarray(on)
        if on.ndim > 1 or on.dtype.kind not in 'biu':
            raise ValueError('on must be a bool / integer scalar or 1-D array')
        if ids is not None:
            if not isinstance(ids, np.ndarray) or ids.ndim != 1:
                raise ValueError('ids must be a 1-D int32 array')
            n = ids.shape[0]
        else:
            n = on.shape[0] if on.ndim == 1 else self.max_streams
        _check_np('ids', ids, np.int32, (n,))
        if on.ndim == 1 and on.shape[0] != n:
            raise ValueError('on has %d entries for %d streams' % (on.shape[0], n))
        flags = np.ascontiguousarray(np.broadcast_to(on != 0, (n,)), dtype=np.uint8)
        check(self.lib.pb_set_stream_history(self._h, _np_ptr(ids), _np_ptr(flags), n))

    def stream_history(self, ids=None) -> np.ndarray:
        """bool array: which of streams ids (host int32 array), or of every stream, have history."""
        n = self.max_streams if ids is None else (ids.shape[0] if isinstance(ids, np.ndarray) and ids.ndim == 1 else -1)
        _check_np('ids', ids, np.int32, (n,))
        out = np.zeros(n, np.uint8)
        check(self.lib.pb_get_stream_history(self._h, _np_ptr(ids), n, _np_ptr(out)))
        return out.astype(bool)

    def read_history(self, ids=None, samples=None, out=None):
        """The last ``samples`` (default: all set_history kept) samples of streams ids, as of the work queued before this call:
        an int16 CUDA tensor [n, samples], oldest first, 0 before the stream's history start and for streams without history.
        ids: int32 CUDA tensor (repeats allowed); None: every stream.  Asynchronous on the current stream."""
        torch = self.torch
        n = ids.numel() if ids is not None else self.max_streams
        self._check_t('ids', ids, torch.int32, n)
        if ids is not None and self.check_ids and n:
            lo, hi = int(ids.min()), int(ids.max())
            if lo < 0 or hi >= self.max_streams:
                raise ValueError('stream ids must lie in [0, %d), got [%d, %d]' % (self.max_streams, lo, hi))
        samples = self._int('samples', self.history_samples if samples is None else samples)
        if out is None:
            out = torch.empty((n, max(samples, 0)), dtype=torch.int16, device=self.device)
        else:
            self._check_t('out', out, torch.int16, n * samples, optional=False)
        check(self.lib.pb_read_history(self._h, _ptr(ids), n, samples, _ptr(out), self._stream()))
        return out

    # ---- recorded corpora
    def corpus_windows(self, n_samples, schedule='listener', chunk=1024) -> int:
        """Windows one recording of n_samples yields under ``schedule`` ('listener' or 'simulate') with chunk ``chunk``."""
        n = int(self.lib.pb_corpus_windows(C.byref(self.cfg), _schedule(schedule), int(chunk), int(n_samples)))
        if n < 0:
            check(n)
        return n

    def _corpus_args(self, pcm, offsets, schedule, chunk):
        """(schedule code, int64 offsets, n_rec, W) of a corpus call, checked."""
        sched = _schedule(schedule)
        offsets, n_rec = self._corpus_recordings(pcm, offsets)
        W = sum(self.corpus_windows(int(L), schedule, chunk) for L in np.diff(offsets))
        return sched, offsets, n_rec, W

    def _corpus_recordings(self, pcm, offsets):
        """(int64 offsets, n_rec) of the recordings of a corpus call, checked."""
        torch = self.torch
        if (not isinstance(pcm, torch.Tensor) or pcm.dtype != torch.int16 or pcm.dim() != 1 or not pcm.is_contiguous()
                or pcm.device != self.device):
            raise ValueError('pcm must be a contiguous 1-D int16 tensor on %s' % self.device)
        offsets = np.asarray(offsets)
        if offsets.ndim != 1 or offsets.shape[0] < 1 or offsets.dtype.kind not in 'iu':
            raise ValueError('offsets must be a 1-D integer array [n_rec + 1]')
        offsets = np.ascontiguousarray(offsets, dtype=np.int64)
        n_rec = offsets.shape[0] - 1
        if n_rec and int(offsets[-1]) > pcm.numel():
            raise ValueError('offsets end at %d, past pcm of %d samples' % (int(offsets[-1]), pcm.numel()))
        lens = np.diff(offsets)
        if lens.size and lens.min() < 0:
            raise ValueError('offsets must be non-decreasing')
        return offsets, n_rec

    def score_corpus(self, pcm, offsets, schedule='listener', chunk=1024, threshold=0.5, divisor=32768):
        """Every bank model over recordings pcm[offsets[r]:offsets[r + 1]] (pcm a 1-D int16 CUDA tensor, offsets a host int64
        array [n_rec + 1]).  Returns dict(raw f32 [M, W], conf f64 [M, W], fired u8 [M, W], activations i64 [M, n_rec], and
        for the simulate schedule above i64 [M, n_rec] and sum f64 [M, n_rec]; None otherwise), W the total window count.
        Asynchronous on the current stream.  Schedules and outputs: pb_score_corpus in include/precise_b200.h."""
        torch = self.torch
        sched, offsets, n_rec, W = self._corpus_args(pcm, offsets, schedule, chunk)
        M = self.num_models
        f = lambda shape, dt: torch.empty(shape, dtype=dt, device=self.device)
        out = dict(raw=f((M, W), torch.float32), conf=f((M, W), torch.float64), fired=f((M, W), torch.uint8),
                   activations=f((M, n_rec), torch.int64), above=None, sum=None)
        if sched == 1:
            out['above'] = f((M, n_rec), torch.int64)
            out['sum'] = f((M, n_rec), torch.float64)
        check(self.lib.pb_score_corpus(self._h, _ptr(pcm), _np_ptr(offsets), n_rec, int(divisor), sched, int(chunk),
                                       float(threshold), _ptr(out['raw']), _ptr(out['conf']), _ptr(out['fired']),
                                       _ptr(out['activations']), _ptr(out['above']), _ptr(out['sum']), self._stream()))
        return out

    def score_corpus_pool(self, pcm, offsets, model_ids, schedule='listener', chunk=1024, threshold=0.5, divisor=32768,
                          per_window=True):
        """Pool models ``model_ids`` (host int32 array [k], repeats allowed) over recordings pcm[offsets[r]:offsets[r + 1]], as
        score_corpus takes them: every model scores every recording, K1 runs once.  Returns score_corpus's dict with k rows in
        the order of model_ids.  per_window=False: raw, conf and fired are None and only the reductions (activations, and
        for the simulate schedule above and sum) are computed, without a [k, W] buffer.  Asynchronous on the current stream.
        pb_score_corpus_pool in include/precise_b200.h."""
        torch = self.torch
        sched, offsets, n_rec, W = self._corpus_args(pcm, offsets, schedule, chunk)
        model_ids = np.asarray(model_ids)
        k = model_ids.shape[0] if model_ids.ndim == 1 else -1
        _check_np('model_ids', model_ids, np.int32, (k,), optional=False)
        f = lambda shape, dt: torch.empty(shape, dtype=dt, device=self.device)
        out = dict(raw=None, conf=None, fired=None, activations=f((k, n_rec), torch.int64), above=None, sum=None)
        if per_window:
            out.update(raw=f((k, W), torch.float32), conf=f((k, W), torch.float64), fired=f((k, W), torch.uint8))
        if sched == 1:
            out['above'] = f((k, n_rec), torch.int64)
            out['sum'] = f((k, n_rec), torch.float64)
        check(self.lib.pb_score_corpus_pool(self._h, _ptr(pcm), _np_ptr(offsets), n_rec, _np_ptr(model_ids), k, int(divisor),
                                            sched, int(chunk), float(threshold), _ptr(out['raw']), _ptr(out['conf']),
                                            _ptr(out['fired']), _ptr(out['activations']), _ptr(out['above']),
                                            _ptr(out['sum']), self._stream()))
        return out

    def score_corpus_pairs(self, pcm, offsets, model_ids, rec_ids, schedule='listener', chunk=1024, threshold=0.5,
                           divisor=32768, per_window=True, hit_threshold=None, hit_capacity=None):
        """Pool model model_ids[p] over recording rec_ids[p] for each pair p (host int32 arrays [n_pairs], repeats and any
        order allowed), recordings as score_corpus takes them.  Returns score_corpus_pool's keys with 1-D pair-major outputs:
        raw, conf, fired [Wp] (pair p's windows at pair_offsets[p] .. pair_offsets[p + 1] - 1; None with per_window=False),
        activations [n_pairs], above and sum [n_pairs] for the simulate schedule, and pair_offsets (host int64 [n_pairs + 1]).
        With a hit_threshold (listener schedule), also hits: the sorted int64 pair-window indices whose conf is above it,
        computed on the device; when more than hit_capacity are found the call runs once more with room for all of them, and
        this (and only this) waits for the device.  pb_score_corpus_pairs in include/precise_b200.h."""
        torch = self.torch
        sched, offsets, n_rec, _ = self._corpus_args(pcm, offsets, schedule, chunk)
        model_ids, rec_ids = np.asarray(model_ids), np.asarray(rec_ids)
        n = model_ids.shape[0] if model_ids.ndim == 1 else -1
        _check_np('model_ids', model_ids, np.int32, (n,), optional=False)
        _check_np('rec_ids', rec_ids, np.int32, (n,), optional=False)
        if n and (rec_ids.min() < 0 or rec_ids.max() >= n_rec):
            raise ValueError('recording ids must lie in [0, %d)' % n_rec)
        counts = np.asarray([self.corpus_windows(int(L), schedule, chunk) for L in np.diff(offsets)], np.int64)
        pw = np.concatenate([[0], np.cumsum(counts[rec_ids], dtype=np.int64)]).astype(np.int64)
        Wp = int(pw[-1])
        f = lambda shape, dt: torch.empty(shape, dtype=dt, device=self.device)
        out = dict(raw=None, conf=None, fired=None, activations=f((n,), torch.int64), above=None, sum=None, pair_offsets=pw)
        if per_window:
            out.update(raw=f((Wp,), torch.float32), conf=f((Wp,), torch.float64), fired=f((Wp,), torch.uint8))
        if sched == 1:
            out['above'] = f((n,), torch.int64)
            out['sum'] = f((n,), torch.float64)
        hits = hit_threshold is not None
        n_hits = f((1,), torch.int64) if hits else None
        cap = self._int('hit_capacity', 1 << 16 if hit_capacity is None else hit_capacity) if hits else 0

        def run(cap):
            d_hits = f((max(cap, 1),), torch.int64) if hits else None
            check(self.lib.pb_score_corpus_pairs(self._h, _ptr(pcm), _np_ptr(offsets), n_rec, _np_ptr(model_ids),
                                                 _np_ptr(rec_ids), n, int(divisor), sched, int(chunk), float(threshold),
                                                 _ptr(out['raw']), _ptr(out['conf']), _ptr(out['fired']),
                                                 _ptr(out['activations']), _ptr(out['above']), _ptr(out['sum']),
                                                 float(hit_threshold) if hits else 0.0, _ptr(d_hits) if cap else None, cap,
                                                 _ptr(n_hits), self._stream()))
            return d_hits

        d_hits = run(cap)
        if hits:
            total = int(n_hits.item())
            if total > cap:
                cap = total
                d_hits = run(cap)
            out['hits'] = torch.sort(d_hits[:total])[0]
        return out

    def score_dataset(self, pcm, offsets, targets, model_ids, rows=None, recs=None, thresholds=(0.5,), divisor=32767,
                      per_entry=True, miss_threshold=None, miss_capacity=None):
        """Pool models over labelled clips pcm[offsets[r]:offsets[r + 1]] (as score_corpus takes recordings; none empty), each
        cropped to its last params.max_samples samples and scored once, as the reference's vectorize + Runner.predict score
        a clip.  targets: host uint8 [n_rec], non-zero = wake word.  model_ids: host int32 [k] pool slots; statistics row i
        belongs to model_ids[i].  rows / recs None: every model over every clip, raw [k, n_rec].  Otherwise host int32
        arrays [n_pairs]: entry p is model_ids[rows[p]] over clip recs[p], raw [n_pairs].  Returns dict(raw (None with
        per_entry=False), count i64 [k, 2], hist i64 [k, 2, 2 n_thr + 1], fit i64 [k, 2, 3], thresholds (the float32 values
        the histogram used)), and with a miss_threshold also misses: the sorted int64 indices (i * n_rec + r, or p) of the
        entries with (raw > miss_threshold) != label; when more than miss_capacity are found the call runs once more with
        room for all of them, and this (and only this) waits for the device.  divisor 32767: clips read as load_audio reads
        wav files.  Asynchronous on the current stream.  pb_score_dataset in include/precise_b200.h."""
        torch = self.torch
        offsets, n_rec = self._corpus_recordings(pcm, offsets)
        targets, model_ids = np.asarray(targets), np.asarray(model_ids)
        _check_np('targets', targets, np.uint8, (n_rec,), optional=False)
        k = model_ids.shape[0] if model_ids.ndim == 1 else -1
        _check_np('model_ids', model_ids, np.int32, (k,), optional=False)
        if (rows is None) != (recs is None):
            raise ValueError('rows and recs come together')
        n = 0
        if rows is not None:
            rows, recs = np.asarray(rows), np.asarray(recs)
            n = rows.shape[0] if rows.ndim == 1 else -1
            _check_np('rows', rows, np.int32, (n,), optional=False)
            _check_np('recs', recs, np.int32, (n,), optional=False)
        thr = np.ascontiguousarray(thresholds, dtype=np.float64)
        if thr.ndim != 1:
            raise ValueError('thresholds must be a 1-D list')
        n_thr = thr.shape[0]
        f = lambda shape, dt: torch.empty(shape, dtype=dt, device=self.device)
        out = dict(raw=None, count=f((k, 2), torch.int64), hist=f((k, 2, 2 * n_thr + 1), torch.int64),
                   fit=f((k, 2, 3), torch.int64), thresholds=thr.astype(np.float32))
        if per_entry:
            out['raw'] = f((n,), torch.float32) if rows is not None else f((k, n_rec), torch.float32)
        misses = miss_threshold is not None
        n_miss = f((1,), torch.int64) if misses else None
        cap = self._int('miss_capacity', 1 << 16 if miss_capacity is None else miss_capacity) if misses else 0

        def run(cap):
            d_miss = f((max(cap, 1),), torch.int64) if misses else None
            check(self.lib.pb_score_dataset(self._h, _ptr(pcm), _np_ptr(offsets), n_rec, _np_ptr(targets), _np_ptr(model_ids), k,
                                            _np_ptr(rows) if n else None, _np_ptr(recs) if n else None, n, int(divisor),
                                            int(self.params.max_samples), _np_ptr(thr), n_thr, _ptr(out['raw']),
                                            _ptr(out['count']), _ptr(out['hist']), _ptr(out['fit']),
                                            float(miss_threshold) if misses else 0.0, _ptr(d_miss) if cap else None, cap,
                                            _ptr(n_miss), self._stream()))
            return d_miss

        if k == 0 or (rows is not None and n == 0):           # no entry (the library reads an empty pair list as "every pair")
            for key in ('count', 'hist', 'fit'):
                out[key].zero_()
            if misses:
                out['misses'] = f((0,), torch.int64)
            return out
        d_miss = run(cap)
        if misses:
            total = int(n_miss.item())
            if total > cap:
                cap = total
                d_miss = run(cap)
            out['misses'] = torch.sort(d_miss[:total])[0]
        return out

    # ---- training (pb_vectorize_clips, pb_train, pb_train_loss)
    def vectorize_clips(self, pcm, offsets, divisor=32767):
        """The network input of each clip pcm[offsets[r]:offsets[r + 1]] (as score_dataset takes them; none empty): float32
        [n_rec, n_features, feature_size] on the device, vectorize(clip) of the last params.max_samples samples, bit for bit
        the window score_dataset scores.  Asynchronous on the current stream.  pb_vectorize_clips in include/precise_b200.h."""
        offsets, n_rec = self._corpus_recordings(pcm, offsets)
        out = self.torch.empty((n_rec, self.n_features, self.feature_size), dtype=self.torch.float32, device=self.device)
        check(self.lib.pb_vectorize_clips(self._h, _ptr(pcm), _np_ptr(offsets), n_rec, int(divisor), int(self.params.max_samples),
                                          _ptr(out), self._stream()))
        return out

    def add_noise(self, pcm, offsets, noise, items, ratios, noise_pos=0, divisor=32767, out=True, inputs=False):
        """Noise from the int16 corpus tensor ``noise`` mixed into clips pcm[offsets[r]:offsets[r + 1]]: item i is clip
        items[i] (int32) with ratio ratios[i] (float64), its noise span read on cyclically from ``noise_pos``.  Returns
        (mixed clips back to back as an int16 tensor, or None with out=False; vectorize of each mixed clip, float32
        [n_items, n_features, feature_size], or None with inputs=False).  Asynchronous on the current stream.  pb_add_noise in
        include/precise_b200.h."""
        torch = self.torch
        offsets, n_rec = self._corpus_recordings(pcm, offsets)
        if (not isinstance(noise, torch.Tensor) or noise.dtype != torch.int16 or noise.dim() != 1 or not noise.is_contiguous()
                or noise.device != self.device):
            raise ValueError('noise must be a contiguous 1-D int16 tensor on %s' % self.device)
        items = np.ascontiguousarray(items, dtype=np.int32)
        ratios = np.ascontiguousarray(ratios, dtype=np.float64)
        n = items.shape[0]
        _check_np('items', items, np.int32, (n,), optional=False)
        _check_np('ratios', ratios, np.float64, (n,), optional=False)
        total = int(np.diff(offsets)[items].sum()) if n and items.min() >= 0 and items.max() < n_rec else 0
        d_out = torch.empty(max(total, 1), dtype=torch.int16, device=self.device) if out else None    # non-null when empty
        d_in = torch.empty((n, self.n_features, self.feature_size), dtype=torch.float32, device=self.device) if inputs else None
        check(self.lib.pb_add_noise(self._h, _ptr(pcm), _np_ptr(offsets), n_rec, _ptr(noise), noise.numel(), _np_ptr(items),
                                    _np_ptr(ratios), n, int(noise_pos), int(divisor), int(self.params.max_samples), _ptr(d_out),
                                    _ptr(d_in), self._stream()))
        return (None if d_out is None else d_out[:total]), d_in

    def generate(self, bg, bg_offsets, clips, clip_offsets, items, segments, windows=None, chunk=2048, divisor=32767, out=True):
        """Clips overlaid on background recordings: backgrounds bg[bg_offsets[b]:bg_offsets[b + 1]] and clips likewise (1-D
        int16 CUDA tensors, host int64 offsets), items a GEN_ITEM array and segments a GEN_SEGMENT array (pb_gen_item /
        pb_gen_segment), windows an int64 array [n_windows, 2] of (item, chunk index) or None.  Returns (the items' streams
        back to back as an int16 tensor, or None with out=False; the windows' network inputs, float32
        [n_windows, n_features, feature_size], or None without windows).  Asynchronous on the current stream.  pb_generate in
        include/precise_b200.h."""
        torch = self.torch
        bg_offsets, n_bg = self._corpus_recordings(bg, bg_offsets)
        clip_offsets, n_clips = self._corpus_recordings(clips, clip_offsets)
        items = np.ascontiguousarray(items, dtype=GEN_ITEM)
        segments = np.ascontiguousarray(segments, dtype=GEN_SEGMENT)
        n = items.shape[0]
        _check_np('items', items, GEN_ITEM, (n,), optional=False)
        _check_np('segments', segments, GEN_SEGMENT, (segments.shape[0],), optional=False)
        if windows is not None:
            windows = np.ascontiguousarray(windows, dtype=np.int64).reshape(-1, 2)
        n_win = 0 if windows is None else windows.shape[0]
        total = int(np.maximum(items['length'], 0).sum())
        d_out = torch.empty(max(total, 1), dtype=torch.int16, device=self.device) if out else None    # non-null when empty
        d_in = (torch.empty((n_win, self.n_features, self.feature_size), dtype=torch.float32, device=self.device)
                if windows is not None else None)
        check(self.lib.pb_generate(self._h, _ptr(bg), _np_ptr(bg_offsets), n_bg, _ptr(clips), _np_ptr(clip_offsets), n_clips,
                                   _np_ptr(items), n, _np_ptr(segments), segments.shape[0],
                                   _np_ptr(windows) if n_win else None, n_win, int(chunk), int(divisor), _ptr(d_out),
                                   _ptr(d_in), self._stream()))
        return (None if d_out is None else d_out[:total]), d_in

    def _train_args(self, inputs, targets, k, rows_of, recs, weights):
        """(n_rec, targets, pair rows, pair recs, n_pairs, stride) of a training call, checked.  The stride is the weight
        rows' width: PB_TRAIN_WIDE_STRIDE (pb_train_wide) when weights holds k rows of it, else PB_TRAIN_STRIDE (pb_train)."""
        torch = self.torch
        if (not isinstance(inputs, torch.Tensor) or inputs.dtype != torch.float32 or not inputs.is_contiguous()
                or inputs.device != self.device or inputs.dim() != 3 or tuple(inputs.shape[1:]) != (self.n_features, self.feature_size)):
            raise ValueError('inputs must be a contiguous float32 tensor [n, %d, %d] on %s' % (self.n_features, self.feature_size,
                                                                                              self.device))
        n_rec = inputs.shape[0]
        targets = np.ascontiguousarray(np.asarray(targets) != 0, dtype=np.uint8)
        if targets.shape != (n_rec,):
            raise ValueError('one target per input')
        wide = k > 0 and isinstance(weights, torch.Tensor) and weights.numel() == k * PB_TRAIN_WIDE_STRIDE
        stride = PB_TRAIN_WIDE_STRIDE if wide else PB_TRAIN_STRIDE
        self._check_t('weights', weights, torch.float32, k * stride, optional=False)
        if (rows_of is None) != (recs is None):
            raise ValueError('rows_of and recs come together')
        if rows_of is None:
            return n_rec, targets, None, None, 0, stride
        pr, pc = np.ascontiguousarray(rows_of, dtype=np.int32), np.ascontiguousarray(recs, dtype=np.int32)
        if pr.ndim != 1 or pr.shape != pc.shape:
            raise ValueError('rows_of and recs must be 1-D arrays of one length')
        return n_rec, targets, pr, pc, pr.shape[0], stride

    @staticmethod
    def train_rows(hidden, activation, recurrent_activation, seed):
        """ctypes array of pb_train_row from per-row lists (activation names as GruModel holds them)."""
        acts = {'linear': 0, 'tanh': 1}
        racts = {'hard_sigmoid': 0, 'sigmoid': 1}
        k = len(hidden)
        arr = (pb_train_row * max(k, 1))()
        for i in range(k):
            arr[i] = pb_train_row(int(hidden[i]), acts[activation[i]], racts[recurrent_activation[i]], int(seed[i]) & 0xFFFFFFFF)
        return arr, k

    def train(self, inputs, targets, rows, weights, rms, rows_of=None, recs=None, epochs=10, epoch0=0, batch_size=5000, lr=0.001,
              rho=0.9, epsilon=1e-7, loss_bias=0.8, dropout=0.2):
        """pb_train: trains the k networks of ``rows`` (train_rows' array) in place in ``weights`` and ``rms`` (float32 CUDA
        tensors [k, PB_TRAIN_STRIDE]) over ``inputs`` (vectorize_clips' tensor) with labels ``targets`` (host, non-zero = wake
        word).  rows_of / recs None: every network on every input; otherwise entry p is input recs[p] of network rows_of[p].
        Returns the float64 epoch losses [k, epochs] (NaN for a network without entries) on the device.  Asynchronous on the
        current stream.  With weights and rms [k, PB_TRAIN_WIDE_STRIDE] the call is pb_train_wide (up to 128 GRU units).
        pb_train and pb_train_wide in include/precise_b200.h."""
        arr, k = rows
        n_rec, targets, pr, pc, n, stride = self._train_args(inputs, targets, k, rows_of, recs, weights)
        self._check_t('rms', rms, self.torch.float32, k * stride, optional=False)
        o = pb_train_opts()
        check(self.lib.pb_train_opts_default(C.byref(o)))
        o.epochs, o.epoch0, o.batch_size = int(epochs), int(epoch0), int(batch_size)
        o.lr, o.rho, o.epsilon, o.loss_bias, o.dropout = lr, rho, epsilon, loss_bias, dropout
        loss = self.torch.empty((k, max(int(epochs), 0)), dtype=self.torch.float64, device=self.device)
        if rows_of is not None and n == 0:                     # no entry (the library reads an empty pair list as "every pair")
            loss.fill_(float('nan'))
            return loss
        fn = self.lib.pb_train_wide if stride == PB_TRAIN_WIDE_STRIDE else self.lib.pb_train
        check(fn(self._h, _ptr(inputs), n_rec, _np_ptr(targets), arr, k, _np_ptr(pr), _np_ptr(pc), n, C.byref(o), _ptr(weights),
                 _ptr(rms), _ptr(loss), self._stream()))
        return loss

    def train_loss(self, inputs, targets, rows, weights, rows_of=None, recs=None, loss_bias=0.8, dropout=0.0, epoch=0, grad=False):
        """pb_train_loss: each network's loss over all its entries as one batch (dropout 0: Keras's evaluate) -> float64
        [k] on the device, and with grad=True also its gradient, float32 [k, stride] (the weights' row width).  Arguments as
        train's; weights [k, PB_TRAIN_WIDE_STRIDE] make it pb_train_wide_loss.  pb_train_loss in include/precise_b200.h."""
        arr, k = rows
        n_rec, targets, pr, pc, n, stride = self._train_args(inputs, targets, k, rows_of, recs, weights)
        torch = self.torch
        loss = torch.empty(k, dtype=torch.float64, device=self.device)
        g = torch.zeros((k, stride), dtype=torch.float32, device=self.device) if grad else None
        if rows_of is not None and n == 0:
            loss.fill_(float('nan'))
            return (loss, g) if grad else loss
        fn = self.lib.pb_train_wide_loss if stride == PB_TRAIN_WIDE_STRIDE else self.lib.pb_train_loss
        check(fn(self._h, _ptr(inputs), n_rec, _np_ptr(targets), arr, k, _np_ptr(pr), _np_ptr(pc), n, float(loss_bias),
                 float(dropout), int(epoch), _ptr(weights), _ptr(loss), _ptr(g), self._stream()))
        return (loss, g) if grad else loss

    def score_rows(self, inputs, targets, rows, weights, pair_rows=None, pair_recs=None, thresholds=(0.5,), per_entry=True,
                   miss_threshold=None, miss_capacity=None):
        """score_dataset's statistics for the k networks of ``rows`` (train_rows' array) given as weight rows ``weights``
        (float32 CUDA tensor [k, stride]: PB_TRAIN_STRIDE up to 24 units, PB_TRAIN_WIDE_STRIDE up to 128, read from its
        width), over ``inputs`` (vectorize_clips' tensor) with labels ``targets`` (host, non-zero = wake word).  pair_rows /
        pair_recs None: every network over every input, raw [k, n_rec]; otherwise entry p is network pair_rows[p] over input
        pair_recs[p], raw [n_pairs].  Returns score_dataset's dict, misses included.  Asynchronous on the current stream (a
        miss list that overflows miss_capacity waits, as in score_dataset).  pb_score_rows in include/precise_b200.h."""
        torch = self.torch
        arr, k = rows
        n_rec, targets, pr, pc, n, stride = self._train_args(inputs, targets, k, pair_rows, pair_recs, weights)
        thr = np.ascontiguousarray(thresholds, dtype=np.float64)
        if thr.ndim != 1:
            raise ValueError('thresholds must be a 1-D list')
        n_thr = thr.shape[0]
        f = lambda shape, dt: torch.empty(shape, dtype=dt, device=self.device)
        out = dict(raw=None, count=f((k, 2), torch.int64), hist=f((k, 2, 2 * n_thr + 1), torch.int64),
                   fit=f((k, 2, 3), torch.int64), thresholds=thr.astype(np.float32))
        if per_entry:
            out['raw'] = f((n,), torch.float32) if pr is not None else f((k, n_rec), torch.float32)
        misses = miss_threshold is not None
        n_miss = f((1,), torch.int64) if misses else None
        cap = self._int('miss_capacity', 1 << 16 if miss_capacity is None else miss_capacity) if misses else 0

        def run(cap):
            d_miss = f((max(cap, 1),), torch.int64) if misses else None
            check(self.lib.pb_score_rows(self._h, _ptr(inputs), n_rec, _np_ptr(targets), arr, k, _ptr(weights), stride,
                                         _np_ptr(pr) if n else None, _np_ptr(pc) if n else None, n, _np_ptr(thr), n_thr,
                                         _ptr(out['raw']), _ptr(out['count']), _ptr(out['hist']), _ptr(out['fit']),
                                         float(miss_threshold) if misses else 0.0, _ptr(d_miss) if cap else None, cap,
                                         _ptr(n_miss), self._stream()))
            return d_miss

        if k == 0 or (pr is not None and n == 0):             # no entry (the library reads an empty pair list as "every pair")
            for key in ('count', 'hist', 'fit'):
                out[key].zero_()
            if misses:
                out['misses'] = f((0,), torch.int64)
            return out
        d_miss = run(cap)
        if misses:
            total = int(n_miss.item())
            if total > cap:
                cap = total
                d_miss = run(cap)
            out['misses'] = torch.sort(d_miss[:total])[0]
        return out

    def rows_groups(self, networks=0, entries=0):
        """Test hook: score_rows splits at most ``networks`` networks per group and scans at most ``entries`` entries per
        batch (whole rows in the cross product); 0 = the default."""
        check(self.lib.pb_debug_rows_groups(self._h, int(networks), int(entries)))

    def corpus_pairs_batch(self, windows):
        """Test hook: score_corpus_pairs scans at most ``windows`` pair-windows per batch (0 = the default)."""
        check(self.lib.pb_debug_corpus_pairs_batch(self._h, int(windows)))

    def corpus_pool_rows(self, rows):
        """Test hook: score_corpus_pool with per_window=False scans at most ``rows`` models per batch (0 = the default)."""
        check(self.lib.pb_debug_corpus_pool_rows(self._h, int(rows)))

    def corpus_pool_scan(self, nm=0, groups_fast=-1):
        """A/B hook: score_corpus_pool's models per CTA (1, 2, 4, 8; 0 = default) and grid order (-1 = default)."""
        check(self.lib.pb_debug_corpus_pool_scan(self._h, int(nm), int(groups_fast)))

    def update_host(self, pcm_np, conf_np, raw_np=None, fired_np=None, ids_np=None) -> int:
        """Host-buffer tick (numpy arrays, ideally backed by pinned memory).  Returns this tick's count."""
        if not isinstance(pcm_np, np.ndarray) or pcm_np.ndim != 2:
            raise ValueError('pcm_np must be an int16 array of shape (n, %d)' % self.chunk_samples)
        n = pcm_np.shape[0]
        _check_np('pcm_np', pcm_np, np.int16, (n, self.chunk_samples), optional=False)
        _check_np('conf_np', conf_np, np.float64, (n,), optional=False)
        _check_np('raw_np', raw_np, np.float32, (n,))
        _check_np('fired_np', fired_np, np.uint8, (n,))
        _check_np('ids_np', ids_np, np.int32, (n,))
        if ids_np is not None and self.check_ids and n:
            if ids_np.min() < 0 or ids_np.max() >= self.max_streams or len(np.unique(ids_np)) != n:
                raise ValueError('stream ids must be unique and lie in [0, %d)' % self.max_streams)
        cnt = C.c_uint64(0)
        vp = _np_ptr
        check(self.lib.pb_update_host(self._h, vp(pcm_np), vp(ids_np), n, vp(raw_np), vp(conf_np), vp(fired_np),
                                      C.cast(C.byref(cnt), C.c_void_p)))
        return int(cnt.value)

    def gru_mode(self, mode):
        check(self.lib.pb_debug_gru_mode(self._h, int(mode)))

    def force_generic(self, on=True):
        check(self.lib.pb_debug_force_generic(self._h, int(on)))

    def k1_mode(self, mode):
        """0 = default MFCC kernel choice (the pipelined FFT kernel on the aligned geometry), 2 = the FFT kernel it replaced
        (bit-identical results), 3 = that kernel with its 64-bit set-up, 4 / 5 / 6 = the DFT on
        mma.sync (stage 2 only / both stages / both stages with a shuffle epilogue)."""
        check(self.lib.pb_debug_k1_mode(self._h, int(mode)))

    # ---- profiling / introspection
    def profile(self, on=True):
        check(self.lib.pb_profile_enable(self._h, int(on)))
        check(self.lib.pb_profile_reset(self._h))

    def profile_read(self):
        ms = (C.c_double * 4)()
        ln = (C.c_uint64 * 4)()
        check(self.lib.pb_profile_read(self._h, ms, ln))
        return list(ms), list(ln)

    def filterbank(self) -> np.ndarray:
        fb = np.zeros((self.params.n_filt, self.params.n_fft // 2 + 1), dtype=np.float64)
        check(self.lib.pb_get_filterbank(self._h, fb.ctypes.data_as(C.c_void_p)))
        return fb

    def cdf(self):
        lo, hi = C.c_int32(), C.c_int32()
        n = self.lib.pb_get_cdf(self._h, None, 0, C.byref(lo), C.byref(hi))
        cd = np.zeros(n, dtype=np.float64)
        self.lib.pb_get_cdf(self._h, cd.ctypes.data_as(C.c_void_p), n, C.byref(lo), C.byref(hi))
        return cd, lo.value, hi.value


def pinned_empty(shape, dtype):
    """numpy array backed by cudaHostAlloc memory (for update_host at PCIe rate)."""
    lib = get_lib()
    dtype = np.dtype(dtype)
    nbytes = int(np.prod(shape)) * dtype.itemsize
    p = C.c_void_p()
    check(lib.pb_host_alloc(C.byref(p), nbytes))
    buf = (C.c_char * max(nbytes, 1)).from_address(p.value)
    arr = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)
    return arr, p


def pinned_free(p):
    check(get_lib().pb_host_free(p))
