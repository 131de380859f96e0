#!/usr/bin/env python3
"""Generate the committed golden fixtures from the REAL reference code.

Needs a checkout of the reference (mycroft-precise, commit e1a635e); the tests only read the committed outputs:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden.py /path/to/mycroft-precise

What is taken from the reference, unmodified, by import:
  * precise.params.ListenerParams            -> params_golden.json
  * precise.threshold_decoder.ThresholdDecoder (+ precise.functions) -> decoder_golden.npz
  * precise_runner.runner.TriggerDetector    -> trigger_golden.npz
  * precise.network_runner.Listener (the real streaming state machine, driven through its
    sanctioned ``runner_cls`` seam, cf. reference precise/scripts/train_generated.py:93)
                                             -> listener_golden.npz

What is NOT from the reference: ``sonopy`` and Keras/TF are absent from this image, so the
Listener is given (a) a ``sonopy`` module whose mfcc_spec/mel_spec delegate to oracle/mfcc.py
and (b) a runner whose predict() is oracle/gru.py.  listener_golden.npz therefore pins the
reference's state machine, decoder and glue around the (unpinned) oracle arithmetic.
"""
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.dont_write_bytecode = True
sys.path.insert(0, ROOT)
REF = os.path.abspath(sys.argv[1])
sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(REF, 'runner'))

sys.path.insert(0, HERE)
from cases import DECODER_CASES, TRIGGER_CASES, LISTENER_CASES, make_pcm   # noqa: E402
from oracle import mfcc as omfcc            # noqa: E402
from oracle import gru as ogru              # noqa: E402

# --- sonopy stand-in: same call signature the reference uses (vectorization.py:32-39) -------
shim = types.ModuleType('sonopy')
shim.mfcc_spec = lambda audio, sample_rate, window_stride=(160, 80), fft_size=512, num_filt=20, \
    num_coeffs=13: omfcc.mfcc_spec(audio, sample_rate, window_stride[0], window_stride[1],
                                   fft_size, num_filt, num_coeffs)
shim.mel_spec = lambda audio, sample_rate, window_stride=(160, 80), fft_size=512, num_filt=20: \
    omfcc.mel_spec(audio, sample_rate, window_stride[0], window_stride[1], fft_size, num_filt)
sys.modules['sonopy'] = shim

from precise.params import ListenerParams, Vectorizer, pr          # noqa: E402
from precise.threshold_decoder import ThresholdDecoder             # noqa: E402
from precise.network_runner import Listener, Runner                # noqa: E402
from precise_runner.runner import TriggerDetector                  # noqa: E402


def params_golden():
    cases = [
        dict(),                                        # reference defaults
        dict(n_mfcc=40, n_filt=40),                    # BASELINE config 3
        dict(buffer_t=2.0, window_t=0.025, hop_t=0.01, n_fft=512),
        dict(sample_rate=8000, window_t=0.064, hop_t=0.032, n_fft=256),
        dict(use_delta=True),
        dict(buffer_t=1.0, window_t=0.03, hop_t=0.0125, n_fft=1024, n_filt=26, n_mfcc=20),
    ]
    base = dict(buffer_t=1.5, window_t=0.1, hop_t=0.05, sample_rate=16000, sample_depth=2,
                n_fft=512, n_filt=20, n_mfcc=13, use_delta=False,
                threshold_config=((6, 4),), threshold_center=0.2, vectorizer=Vectorizer.mfccs)
    out = []
    for c in cases:
        kw = dict(base, **c)
        p = ListenerParams(**kw)
        out.append(dict(
            fields={k: (list(map(list, v)) if k == 'threshold_config' else v) for k, v in kw.items()},
            derived=dict(window_samples=p.window_samples, hop_samples=p.hop_samples,
                         buffer_samples=p.buffer_samples, n_features=p.n_features,
                         max_samples=p.max_samples, feature_size=p.feature_size)))
    with open(os.path.join(HERE, 'params_golden.json'), 'w') as f:
        json.dump(out, f, indent=1)


def decoder_golden():
    rs = np.random.RandomState(7)
    logits = np.concatenate([rs.uniform(-30, 30, 4000), rs.randn(2000) * 3, np.linspace(-12, 24, 997)])
    raws32 = (1.0 / (1.0 + np.exp(-logits.astype(np.float32)))).astype(np.float32)
    raws32 = np.concatenate([raws32, np.float32([0.0, 1.0, 0.5, 0.9, 0.99, 0.999, 1e-30, 1 - 2 ** -24])])
    out = {'raws': raws32}
    for i, (cfg, center) in enumerate(DECODER_CASES):
        d = ThresholdDecoder(cfg, center)
        out['cd_%d' % i] = np.asarray(d.cd, dtype=np.float64)
        out['meta_%d' % i] = np.array([d.min_out, d.max_out, d.out_range], dtype=np.int64)
        out['dec_%d' % i] = np.array([d.decode(float(r)) for r in raws32], dtype=np.float64)
        # what Listener.update really passes: the np.float32 scalar Runner.run returns (network_runner.py:73-74, :153).
        # Under this image's NumPy (>= 2) `1 / x - 1` in functions.asigmoid then stays float32; dec_* above is the
        # float64 evaluation (python float in, which is also what NumPy 1.16 promotion gives for np.float32 in).
        with np.errstate(all='ignore'):
            out['dec32_%d' % i] = np.array([d.decode(r) for r in raws32], dtype=np.float64)
        if d.out_range:
            out['enc_%d' % i] = np.array([d.encode(t) for t in np.linspace(0.02, 0.98, 49)], dtype=np.float64)
    out['kat'] = np.array([ThresholdDecoder(((6, 4),), 0.2).decode(v) for v in (0.0, 1.0, 0.5, 0.9, 0.99, 0.999)])
    np.savez_compressed(os.path.join(HERE, 'decoder_golden.npz'), **out)


def trigger_golden():
    rs = np.random.RandomState(11)
    out = {}
    for i, (chunk, sens, lvl) in enumerate(TRIGGER_CASES):
        # bursty probabilities: runs of high and low values
        probs = []
        while len(probs) < 600:
            n = rs.randint(1, 14)
            hi = rs.rand() < 0.45
            probs += list(rs.uniform(0.55, 1.0, n) if hi else rs.uniform(0.0, 0.6, n))
        probs = np.array(probs[:600])
        det = TriggerDetector(chunk, sens, lvl)
        fired, act = [], []
        for p in probs:
            fired.append(det.update(float(p)))
            act.append(det.activation)
        out['probs_%d' % i] = probs
        out['fired_%d' % i] = np.array(fired, dtype=bool)
        out['act_%d' % i] = np.array(act, dtype=np.int64)
        out['cfg_%d' % i] = np.array([chunk, sens, lvl], dtype=np.float64)
    det = TriggerDetector(2048, 0.5, 3)
    out['kat'] = np.array([det.update(p) for p in [0.9] * 6 + [0.1] * 3 + [0.9] * 10], dtype=bool)
    np.savez_compressed(os.path.join(HERE, 'trigger_golden.npz'), **out)


def listener_golden(scale=0.3, fname='listener_golden.npz'):
    weights = ogru.GruWeights.random(13, 20, seed=0, scale=scale)

    class OracleRunner(Runner):
        def __init__(self, _):
            pass

        def predict(self, inputs):
            return ogru.predict(weights, inputs)

        def run(self, inp):
            return self.predict(inp[np.newaxis])[0][0]

    out = {'kernel': weights.kernel, 'recurrent': weights.recurrent, 'bias': weights.bias,
           'dense_w': weights.dense_w, 'dense_b': np.float32(weights.dense_b)}
    for i, (kind, chunk, n_chunks) in enumerate(LISTENER_CASES):
        pcm = make_pcm(100 + i, chunk * n_chunks, kind)
        lis = Listener('', chunk * 2, runner_cls=OracleRunner)
        confs, rings = [], []
        for k in range(n_chunks):
            a = pcm[k * chunk:(k + 1) * chunk].astype(np.float32) / 32768.0   # == buffer_to_audio(bytes)
            confs.append(lis.update(a))
            rings.append(lis.mfccs.copy())
        out['pcm_%d' % i] = pcm
        out['chunk_%d' % i] = np.int64(chunk)
        out['conf_%d' % i] = np.array(confs, dtype=np.float64)
        out['ring_%d' % i] = np.array(rings, dtype=np.float64)[::5]      # every 5th window, keeps it small
        out['carry_%d' % i] = np.int64(len(lis.window_audio))
    out['numpy_version'] = np.array(np.__version__)
    np.savez_compressed(os.path.join(HERE, fname), **out)


if __name__ == '__main__':
    assert pr.window_samples == 1600 and pr.hop_samples == 800 and pr.n_features == 29
    params_golden()
    decoder_golden()
    trigger_golden()
    listener_golden()
    # well-conditioned weights (outputs away from saturation): the set the tight end-to-end assertions use
    listener_golden(scale=0.1, fname='listener_golden_s01.npz')
    for f in sorted(os.listdir(HERE)):
        print(f, os.path.getsize(os.path.join(HERE, f)))
