"""``precise-train`` on the GPU (reference: precise/scripts/train.py, precise/model.py:57-91) for several networks on one
folder of labelled clips.

    python -m mycroft_precise_b200.train MODEL.npz [MODEL.npz ...] FOLDER [-e EPOCHS] [-b BATCH] [-s SENSITIVITY]
                                         [--dropout RATE] [--seed SEED] [--hidden UNITS]

FOLDER has TrainData.from_folder's layout, as precise-test reads it (test.load_folder): the clips under ``FOLDER/wake-word``
and ``FOLDER/not-wake-word`` are trained on, and those under ``FOLDER/test/...`` give the val_loss.  An existing MODEL.npz
(with its .params) is fine-tuned; a missing one is created with GruModel.init (``--hidden`` units, seed ``--seed`` + i for
the i-th model) at the default ListenerParams.  Every model must share the first one's front end and be of the fused family
(hidden <= 24, feature size <= 16, no deltas); all of them train at once in one set of device calls (offline.train).  For
each model, in the order given, a ``=== <model file> ===`` heading is printed, then one line per epoch with its loss and
val_loss as Keras prints them.  Each model's weights are saved to its .npz and its .params written next to it.
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
    ap.add_argument('--hidden', type=int, default=20, help='GRU units of new networks')
    ap.add_argument('--device', type=int, default=0)
    args = ap.parse_args(argv)

    from .core import PreciseB200
    from .model_io import GruModel, load_weights, save_weights
    from .offline import TrainState, train, vectorize_clips
    from .params import ListenerParams, load_params, save_params
    from .simulate import check_pool_models
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
    check_pool_models(names, models)
    pr = models[0][1]
    _, clips, targets = load_folder(args.folder, True, pr.sample_rate)
    _, v_clips, v_targets = load_folder(args.folder, False, pr.sample_rate)
    if not clips:
        raise SystemExit('no training clips under %s' % args.folder)
    core = PreciseB200(pr, hidden=models[0][0].hidden, device=args.device, activation=models[0][0].activation,
                       recurrent_activation=models[0][0].recurrent_activation)
    inputs = vectorize_clips(core, clips)
    state = TrainState.from_models(core, [m for m, _ in models], [args.seed + i for i in range(len(models))])
    kw = dict(epochs=args.epochs, batch_size=args.batch_size, sensitivity=args.sensitivity, dropout=args.dropout)
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
