"""``precise-train-generated`` on the GPU (reference: precise/scripts/train_generated.py) for several networks at once:
wake words overlaid on background recordings, generated and labelled on the device every epoch.

    python -m mycroft_precise_b200.train_generated MODEL.npz [MODEL.npz ...] FOLDER -r RANDOM_FOLDER [-e EPOCHS]
                                                   [-b BATCH] [-t STEPS] [-c CHUNK] [-s SENSITIVITY] [--dropout RATE]
                                                   [--seed SEED] [--hidden UNITS] [-sb] [-p SAVE_PROB]

FOLDER has TrainData.from_folder's layout, as train reads it: the clips under FOLDER/wake-word and FOLDER/not-wake-word are
overlaid (each list sorted by path and cycled), and those under FOLDER/test/... give the val_loss.  RANDOM_FOLDER's wavs
(searched recursively, sorted) are the backgrounds.  Models are created or fine-tuned as train does them, with up to 128 GRU
units (feature size <= 16, no deltas).  Each epoch is
STEPS x BATCH generated windows (offline.Generator, keyed by --seed) and one training epoch over them (pb_train shuffles
them, where Keras's fit_generator takes consecutive batches).  Per model a ``=== <model file> ===`` heading and one
Keras-style line per epoch are printed.  The weights go to each .npz (with -sb only when the epoch's loss is the model's best
so far, as ModelCheckpoint(save_best_only) monitors loss), the .params next to it, and the epochs done to <model>.epoch,
from which a later run resumes (the generator replays to that epoch).  -p saves each window with probability SAVE_PROB as
debug/ww or debug/nww/'<background> - <chunk>.wav': the buffer_samples generated samples that end at it.
"""
import argparse
import fnmatch
import os

import numpy as np


def find_backgrounds(folder: str):
    out = []
    for root, _, names in os.walk(folder):
        out += [os.path.join(root, n) for n in fnmatch.filter(names, '*.wav')]
    return sorted(out)


def read_epoch(model: str) -> int:
    """The reference's Fitipy counter: <model without extension>.epoch, 0 when missing."""
    p = os.path.splitext(model)[0] + '.epoch'
    if not os.path.isfile(p):
        return 0
    with open(p) as f:
        text = f.read().strip()
    return int(text) if text else 0


def write_epoch(model: str, epoch: int):
    with open(os.path.splitext(model)[0] + '.epoch', 'w') as f:
        f.write(str(int(epoch)))


def main(argv=None):
    ap = argparse.ArgumentParser(prog='precise-train-generated', description=__doc__,
                                 formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('model', nargs='+', help='weights file(s) (.npz) to fine-tune or create')
    ap.add_argument('folder', help='folder with wake-word / not-wake-word clips (and test/ with the same)')
    ap.add_argument('-r', '--random-data-folder', default='data/random', help='folder of background wavs')
    ap.add_argument('-e', '--epochs', type=int, default=100, help='number of epochs to train on')
    ap.add_argument('-b', '--batch-size', type=int, default=200, help='number of samples in each batch')
    ap.add_argument('-t', '--steps-per-epoch', type=int, default=100, help='number of steps that are considered an epoch')
    ap.add_argument('-c', '--chunk-size', type=int, default=2048, help='audio samples between generated samples')
    ap.add_argument('-s', '--sensitivity', type=float, default=0.2, help='weighted loss bias: higher = more false negatives')
    ap.add_argument('--dropout', type=float, default=0.2, help='input dropout rate of the GRU')
    ap.add_argument('--seed', type=int, default=0, help='seed of new networks (seed + i), of the generator and of every shuffle')
    ap.add_argument('--hidden', type=int, default=20, help='GRU units of new networks (1 to 128)')
    ap.add_argument('-sb', '--save-best', action='store_true', help="save a model only when its epoch's loss improves")
    ap.add_argument('-p', '--save-prob', type=float, default=0.0, help='probability of saving a window into debug/ww or debug/nww')
    ap.add_argument('--device', type=int, default=0)
    args = ap.parse_args(argv)

    from .core import PreciseB200
    from .model_io import GruModel, load_weights, save_weights
    from .offline import Generator, TrainState, train_generated, vectorize_clips
    from .params import ListenerParams, load_params, save_params
    from .simulate import check_train_models, read_wav
    from .test import find_wavs, load_folder
    names = args.model
    for n in names:
        if not n.endswith('.npz'):
            raise ValueError('%s: the trained networks are written as .npz' % n)
    epochs0 = {read_epoch(n) for n in names}
    if len(epochs0) != 1:
        raise SystemExit('the models have different .epoch counters %s: train them separately' % sorted(epochs0))
    epoch0 = epochs0.pop()
    models = []
    for i, n in enumerate(names):
        if os.path.isfile(n):
            models.append((load_weights(n), load_params(n)))
        else:
            pr = ListenerParams()
            models.append((GruModel.init(pr.feature_size, args.hidden, args.seed + i), pr))
    check_train_models(names, models)
    pr = models[0][1]
    ww, nww = (sorted(f) for f in find_wavs(args.folder))
    wake = [read_wav(f, pr.sample_rate) for f in ww]
    other = [read_wav(f, pr.sample_rate) for f in nww]
    bg_files = find_backgrounds(args.random_data_folder)
    backgrounds = [read_wav(f, pr.sample_rate) for f in bg_files]
    if not wake or not other:
        raise SystemExit('the generator needs wake-word and not-wake-word clips under %s' % args.folder)
    if not backgrounds:
        raise SystemExit('no background wavs under %s' % args.random_data_folder)
    _, v_clips, v_targets = load_folder(args.folder, False, pr.sample_rate)
    core = PreciseB200(pr, hidden=models[0][0].hidden, device=args.device, activation=models[0][0].activation,
                       recurrent_activation=models[0][0].recurrent_activation)
    gen = Generator(core, backgrounds, wake, other, chunk=args.chunk_size, seed=args.seed, names=bg_files)
    state = TrainState.from_models(core, [m for m, _ in models], [args.seed + i for i in range(len(models))])
    state.epoch = epoch0
    validation = (vectorize_clips(core, v_clips), v_targets) if v_clips else None
    kw = dict(steps_per_epoch=args.steps_per_epoch, batch_size=args.batch_size, sensitivity=args.sensitivity,
              dropout=args.dropout, validation=validation, save_prob=args.save_prob)
    k = len(names)
    loss, val, best = np.zeros((k, 0)), np.zeros((k, 0)), np.full(k, np.inf)
    for _ in range(args.epochs):
        res = train_generated(core, state, gen, 1, **kw)
        l, v = res if validation is not None else (res, None)
        loss = np.concatenate([loss, l], 1)
        if v is not None:
            val = np.concatenate([val, v], 1)
        for i, (name, m) in enumerate(zip(names, state.models())):
            if not args.save_best or l[i, 0] < best[i]:
                best[i] = min(best[i], l[i, 0])
                save_weights(name, m)
                save_params(name, models[i][1])
            write_epoch(name, state.epoch)
    for i, name in enumerate(names):
        print('=== %s ===' % name)
        for e in range(args.epochs):
            line = 'Epoch %d/%d - loss: %.4f' % (epoch0 + e + 1, epoch0 + args.epochs, loss[i, e])
            if validation is not None:
                line += ' - val_loss: %.4f' % val[i, e]
            print(line)
    core.close()
    return loss


if __name__ == '__main__':
    main()
