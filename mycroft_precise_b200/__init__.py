"""mycroft_precise_b200 -- H100 (sm_90a) implementation of Mycroft Precise's streaming-inference
hot path (MFCC -> GRU window scan -> threshold decode -> trigger) behind the reference's own
interfaces.  The compute lives in csrc/libprecise_b200.so (hand-written CUDA, C ABI declared in
include/precise_b200.h); this package is the thin Python host that mirrors

    precise.network_runner.Runner / Listener        -> B200Runner / B200Listener
    precise_runner.runner.Engine                     -> B200Engine
    precise/scripts/engine.py (precise-engine)       -> python -m mycroft_precise_b200.engine
    (new) many streams per call                      -> StreamBatch

There is no CPU fallback: importing works anywhere, any compute call needs the built library and
a CUDA device and raises otherwise.
"""
from .params import ListenerParams, Vectorizer, load_params      # noqa: F401
from .core import PreciseB200, PBError, lib_path                 # noqa: F401
from .runner import B200Runner, B200Listener, B200Engine, Engine, TriggerDetector  # noqa: F401
from .batch import StreamBatch                                    # noqa: F401
from .model_io import load_weights, save_weights, GruModel        # noqa: F401
from . import offline                                             # noqa: F401

__version__ = '0.1.0'
