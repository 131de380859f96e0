"""``precise-train`` on the GPU (reference: precise/scripts/train.py, precise/model.py:57-91) for several networks on one
folder of labelled clips.

    python -m mycroft_precise_b200.train MODEL.npz [MODEL.npz ...] FOLDER [-e EPOCHS] [-b BATCH] [-s SENSITIVITY]
                                         [--dropout RATE] [--seed SEED] [--hidden UNITS]
                                         [--noise-folder NOISE_FOLDER [-if N] [-nl LOW] [-nh HIGH]]

FOLDER has TrainData.from_folder's layout, as precise-test reads it (test.load_folder): the clips under ``FOLDER/wake-word``
and ``FOLDER/not-wake-word`` are trained on, and those under ``FOLDER/test/...`` give the val_loss.  An existing MODEL.npz
(with its .params) is fine-tuned; a missing one is created with GruModel.init (``--hidden`` units, seed ``--seed`` + i for
the i-th model) at the default ListenerParams.  Every model must share the first one's front end (feature size <= 16, no
deltas) and have at most 128 GRU units; all of them train at once in one set of device calls (offline.train: pb_train when
every model has at most 24 units, pb_train_wide on the tensor cores when any has more).  For
each model, in the order given, a ``=== <model file> ===`` heading is printed, then one line per epoch with its loss and
val_loss as Keras prints them.  Each model's weights are saved to its .npz and its .params written next to it.

With ``--noise-folder``, every epoch also trains on N fresh noisy copies of each training clip (offline.Augment): noise from
NOISE_FOLDER/*.wav (sorted, read as one cyclic stream, as precise-add-noise reads it) at ratios between LOW and HIGH drawn
from ``--seed``.  The validation clips stay clean.
"""
import argparse
import os

import numpy as np


def main(argv=None):
    ap = argparse.ArgumentParser(prog='precise-train', description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('model', nargs='+', help='weights file(s) (.npz) to fine-tune or create')
    ap.add_argument('folder', help='folder with wake-word / not-wake-word clips (and test/ with the same)')
    ap.add_argument('-e', '--epochs', type=int, default=10, help='number of epochs to train for')
    ap.add_argument('-b', '--batch-size', type=int, default=5000, help='batch size for training')
    ap.add_argument('-s', '--sensitivity', type=float, default=0.2, help='weighted loss bias: higher = more false negatives')
    ap.add_argument('--dropout', type=float, default=0.2, help='input dropout rate of the GRU')
    ap.add_argument('--seed', type=int, default=0, help='seed of new networks (seed + i) and of every shuffle and mask')
    ap.add_argument('--hidden', type=int, default=20, help='GRU units of new networks (1 to 128)')
    ap.add_argument('--device', type=int, default=0)
    ap.add_argument('--noise-folder', default=None, help='folder of noise wavs: train on fresh noisy copies every epoch')
    ap.add_argument('-if', '--inflation-factor', type=int, default=1, help='noisy copies of each clip per epoch')
    ap.add_argument('-nl', '--noise-ratio-low', type=float, default=0.0, help='minimum ratio of noise to sample')
    ap.add_argument('-nh', '--noise-ratio-high', type=float, default=0.4, help='maximum ratio of noise to sample')
    args = ap.parse_args(argv)

    from .core import PreciseB200
    from .model_io import GruModel, load_weights, save_weights
    from .offline import TrainState, train, vectorize_clips
    from .params import ListenerParams, load_params, save_params
    from .simulate import check_train_models
    from .test import load_folder
    names = args.model
    for n in names:
        if not n.endswith('.npz'):
            raise ValueError('%s: the trained networks are written as .npz' % n)
    models = []
    for i, n in enumerate(names):
        if os.path.isfile(n):
            models.append((load_weights(n), load_params(n)))
        else:
            pr = ListenerParams()
            models.append((GruModel.init(pr.feature_size, args.hidden, args.seed + i), pr))
    check_train_models(names, models)
    pr = models[0][1]
    _, clips, targets = load_folder(args.folder, True, pr.sample_rate)
    _, v_clips, v_targets = load_folder(args.folder, False, pr.sample_rate)
    if not clips:
        raise SystemExit('no training clips under %s' % args.folder)
    core = PreciseB200(pr, hidden=models[0][0].hidden, device=args.device, activation=models[0][0].activation,
                       recurrent_activation=models[0][0].recurrent_activation)
    state = TrainState.from_models(core, [m for m, _ in models], [args.seed + i for i in range(len(models))])
    kw = dict(epochs=args.epochs, batch_size=args.batch_size, sensitivity=args.sensitivity, dropout=args.dropout)
    if args.noise_folder is None:
        inputs = vectorize_clips(core, clips)
    else:
        import glob
        from .offline import Augment, NoiseSource
        from .simulate import read_wav
        noise = [read_wav(f, pr.sample_rate) for f in sorted(glob.glob(os.path.join(args.noise_folder, '*.wav')))]
        if sum(n.shape[0] for n in noise) == 0:
            raise SystemExit('no noise audio in %s/*.wav' % args.noise_folder)
        inputs = clips
        kw['augment'] = Augment(NoiseSource(core, noise), args.inflation_factor, args.noise_ratio_low, args.noise_ratio_high,
                                args.seed)
    if v_clips:
        loss, val = train(core, state, inputs, targets, validation=(vectorize_clips(core, v_clips), v_targets), **kw)
    else:
        loss, val = train(core, state, inputs, targets, **kw), None
    for i, (name, m) in enumerate(zip(names, state.models())):
        print('=== %s ===' % name)
        for e in range(args.epochs):
            line = 'Epoch %d/%d - loss: %.4f' % (e + 1, args.epochs, loss[i, e])
            if val is not None:
                line += ' - val_loss: %.4f' % val[i, e]
            print(line)
        save_weights(name, m)
        save_params(name, models[i][1])
    core.close()
    return np.asarray(loss)


if __name__ == '__main__':
    main()
