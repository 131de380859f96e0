"""``precise-simulate`` on the GPU (reference: precise/scripts/simulate.py): false-activation metrics of a model over a
folder of long recordings.

    python -m mycroft_precise_b200.simulate MODEL [MODEL ...] FOLDER [-c CHUNK_SIZE] [-t THRESHOLD]

Every ``*.wav`` of FOLDER (glob order, as the reference) is read as load_audio reads it (precise/util.py:55-72): 16-bit
PCM at the model's sample rate, samples / 32767; a file the wave module cannot parse counts as empty and is skipped; any
other sample width or rate raises.  All files are scored in one batch on the device (offline.simulate), then each file's
metric block and the Total block are printed in the reference's format.  The reference's progress lines (MFCCs... /
Splitting... / Predicting...) are not printed.  A file too short for one window counts its hours with no windows; the
reference fails on it.

With two or more models, every model must share the first one's front end and be of the fused family (hidden <= 24,
feature size <= 16, no deltas).  They are loaded into a model pool and scored together over one MFCC pass
(offline.simulate_pool); for each model, in the order given, a ``=== <model file> ===`` heading is printed, then that
model's per-file blocks and its Total block.
"""
import argparse
import wave
from glob import glob
from os.path import basename, join

import numpy as np


class InvalidAudio(ValueError):
    pass


def read_wav(path: str, sample_rate: int = 16000) -> np.ndarray:
    """int16 mono samples of a wav file under load_audio's rules; an unreadable file gives an empty array."""
    try:
        with wave.open(path, 'rb') as w:
            width, rate, channels = w.getsampwidth(), w.getframerate(), w.getnchannels()
            data = w.readframes(w.getnframes())
    except (EOFError, wave.Error):
        return np.zeros(0, np.int16)
    if width != 2:
        raise InvalidAudio('Unsupported data type: %d-byte samples' % width)
    if rate != sample_rate:
        raise InvalidAudio('Unsupported sample rate: ' + str(rate))
    if channels != 1:
        raise InvalidAudio('Unsupported channel count: ' + str(channels))
    return np.frombuffer(data[:len(data) & ~1], dtype='<i2').astype(np.int16)


def main(argv=None):
    ap = argparse.ArgumentParser(prog='precise-simulate', description=__doc__,
                                 formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('model', nargs='+', help='weights file(s) (.npz, .net or .pb) with their .params next to them')
    ap.add_argument('folder', help='folder with a set of long wav files to test against')
    ap.add_argument('-c', '--chunk_size', type=int, default=4096, help='number of samples between tests')
    ap.add_argument('-t', '--threshold', type=float, default=0.5, help='network output required to be considered an activation')
    ap.add_argument('--device', type=int, default=0)
    args = ap.parse_args(argv)

    from .core import PreciseB200
    from .params import ListenerParams
    from .runner import _resolve_model
    models = [_resolve_model(m) for m in args.model]
    models = [(model, pr or ListenerParams()) for model, pr in models]
    if len(models) > 1:
        check_pool_models(args.model, models)
    model, pr = models[0]
    core = PreciseB200(pr, hidden=model.hidden, device=args.device, activation=model.activation,
                       recurrent_activation=model.recurrent_activation)
    files = glob(join(args.folder, '*.wav'))
    audio = [read_wav(f, pr.sample_rate) for f in files]
    if len(models) == 1:
        from .offline import simulate
        core.load_weights(model.kernel, model.recurrent, model.bias, model.dense_w, model.dense_b)
        metrics, total = simulate(core, audio, args.chunk_size, args.threshold)
        print_metrics(files, metrics, total)
    else:
        from .offline import simulate_pool
        core.set_pool(len(models))
        for i, (m, p) in enumerate(models):
            core.pool_load(i, m, p)
        metrics, totals = simulate_pool(core, audio, np.arange(len(models), dtype=np.int32), args.chunk_size, args.threshold)
        for name, ms, total in zip(args.model, metrics, totals):
            print()
            print('=== %s ===' % name)
            print_metrics(files, ms, total)
    core.close()


def check_pool_models(names, models):
    """Two or more models are scored as one pool: each must share the first one's front end and be of the fused family."""
    from .core import FRONT_END_FIELDS
    pr0 = models[0][1]
    for name, (model, pr) in zip(names, models):
        diff = [f for f in FRONT_END_FIELDS if getattr(pr, f) != getattr(pr0, f)]
        if diff:
            raise ValueError('%s: front end differs from %s in %s; models scored together share one MFCC front end'
                             % (name, names[0], ', '.join(diff)))
        if model.hidden > 24 or model.feature_size > 16 or pr.use_delta:
            raise ValueError('%s: only networks of the fused family (hidden <= 24, feature size <= 16, no deltas) can be '
                             'scored together; this one has hidden = %d, feature size = %d%s'
                             % (name, model.hidden, model.feature_size, ', deltas' if pr.use_delta else ''))


def check_train_models(names, models):
    """Networks trained together: each must share the first one's front end, which training covers for feature size <= 16
    without deltas, and have at most 128 units (pb_train up to 24, pb_train_wide beyond)."""
    from .core import FRONT_END_FIELDS
    pr0 = models[0][1]
    for name, (model, pr) in zip(names, models):
        diff = [f for f in FRONT_END_FIELDS if getattr(pr, f) != getattr(pr0, f)]
        if diff:
            raise ValueError('%s: front end differs from %s in %s; models trained together share one MFCC front end'
                             % (name, names[0], ', '.join(diff)))
        if model.hidden > 128 or model.feature_size > 16 or pr.use_delta:
            raise ValueError('%s: training covers hidden <= 128, feature size <= 16 and no deltas; this one has hidden = %d, '
                             'feature size = %d%s' % (name, model.hidden, model.feature_size, ', deltas' if pr.use_delta else ''))


def print_metrics(files, metrics, total):
    for f, m in zip(files, metrics):
        if m is None:
            continue
        print()
        print(m.info_string(basename(f)))
    print()
    print()
    print(total.info_string('Total'))


if __name__ == '__main__':
    main()
