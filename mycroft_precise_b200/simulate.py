"""``precise-simulate`` on the GPU (reference: precise/scripts/simulate.py): false-activation metrics of a model over a
folder of long recordings.

    python -m mycroft_precise_b200.simulate MODEL FOLDER [-c CHUNK_SIZE] [-t THRESHOLD]

Every ``*.wav`` of FOLDER (glob order, as the reference) is read as load_audio reads it (precise/util.py:55-72): 16-bit
PCM at the model's sample rate, samples / 32767; a file the wave module cannot parse counts as empty and is skipped; any
other sample width or rate raises.  All files are scored in one batch on the device (offline.simulate), then each file's
metric block and the Total block are printed in the reference's format.  The reference's progress lines (MFCCs... /
Splitting... / Predicting...) are not printed.  A file too short for one window counts its hours with no windows; the
reference fails on it.
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
    ap.add_argument('model', help='weights file (.npz, .net or .pb) with its .params next to it')
    ap.add_argument('folder', help='folder with a set of long wav files to test against')
    ap.add_argument('-c', '--chunk_size', type=int, default=4096, help='number of samples between tests')
    ap.add_argument('-t', '--threshold', type=float, default=0.5, help='network output required to be considered an activation')
    ap.add_argument('--device', type=int, default=0)
    args = ap.parse_args(argv)

    from .core import PreciseB200
    from .offline import simulate
    from .params import ListenerParams
    from .runner import _resolve_model
    model, pr = _resolve_model(args.model)
    pr = pr or ListenerParams()
    core = PreciseB200(pr, hidden=model.hidden, device=args.device, activation=model.activation,
                       recurrent_activation=model.recurrent_activation)
    core.load_weights(model.kernel, model.recurrent, model.bias, model.dense_w, model.dense_b)
    files = glob(join(args.folder, '*.wav'))
    audio = [read_wav(f, pr.sample_rate) for f in files]
    metrics, total = simulate(core, audio, args.chunk_size, args.threshold)
    for f, m in zip(files, metrics):
        if m is None:
            continue
        print()
        print(m.info_string(basename(f)))
    print()
    print()
    print(total.info_string('Total'))
    core.close()


if __name__ == '__main__':
    main()
