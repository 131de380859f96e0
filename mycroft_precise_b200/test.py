"""``precise-test`` on the GPU (reference: precise/scripts/test.py, precise/stats.py): a model's true / false positives and
negatives over a folder of labelled clips.

    python -m mycroft_precise_b200.test MODEL [MODEL ...] FOLDER [-u] [-t THRESHOLD] [-nf] [--calc-threshold]

FOLDER has TrainData.from_folder's layout (precise/train_data.py:53-67): ``FOLDER/test/wake-word`` and
``FOLDER/test/not-wake-word`` are tested, or with ``-u`` the training clips ``FOLDER/wake-word`` and
``FOLDER/not-wake-word``; ``*.wav`` is searched recursively, as glob_all does.  Every clip is read as load_audio reads it
(simulate.read_wav: 16-bit mono PCM at the model's sample rate, samples / 32767); an empty or unreadable file is skipped.
Each clip is scored once, on its last buffer_t seconds, as the reference's vectorize + Runner.predict score it.

Every model must share the first one's front end.  When all are of the fused family (hidden <= 24, feature size <= 16, no
deltas), they are loaded into one model pool and scored over the clips in one pass (offline.test_pool).  When any has more
than 24 units, every model must have at most 128 units, feature size <= 16 and no deltas: the clips are vectorized once
(offline.vectorize_clips), the networks packed as weight rows (offline.TrainState.from_models) and scored from them in one
pass (offline.test_rows).  Both print the same blocks.  For each model,
in the order given, a ``=== <model file> ===`` heading is printed, then (unless ``-nf``) the false-positive and
false-negative file lists, then Stats.counts_str and Stats.summary_str as precise-test prints them.  With
``--calc-threshold`` the ``Peak: ... mu, ... std`` line of precise-calc-threshold follows (offline.calc_threshold); the
model's .params file is not written.  The reference's ``Data:`` line is not printed.
"""
import argparse
import fnmatch
import os
from os.path import join

import numpy as np


def find_wavs(folder: str):
    """(wake-word files, not-wake-word files) of ``folder``, searched as precise/util.py:96-110 searches them."""
    def walk(sub):
        out = []
        for root, _, names in os.walk(join(folder, sub)):
            out += [join(root, n) for n in fnmatch.filter(names, '*.wav')]
        return out
    return walk('wake-word'), walk('not-wake-word')


def load_folder(folder: str, use_train: bool, sample_rate: int = 16000):
    """(files, clips, targets) of the folder's test (or training) set, wake-word clips first; empty files are left out."""
    from .simulate import read_wav
    ww, nww = find_wavs(folder if use_train else join(folder, 'test'))
    files, clips, targets = [], [], []
    for f, t in [(f, 1) for f in ww] + [(f, 0) for f in nww]:
        a = read_wav(f, sample_rate)
        if a.shape[0] == 0:
            continue
        files.append(f)
        clips.append(a)
        targets.append(t)
    return files, clips, np.asarray(targets, np.uint8)


def main(argv=None):
    ap = argparse.ArgumentParser(prog='precise-test', description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('model', nargs='+', help='weights file(s) (.npz, .net or .pb) with their .params next to them')
    ap.add_argument('folder', help='folder with wake-word / not-wake-word clips (and test/ with the same)')
    ap.add_argument('-u', '--use-train', action='store_true', help='evaluate training data instead of test data')
    ap.add_argument('-nf', '--no-filenames', action='store_true', help="don't print out the names of files that failed")
    ap.add_argument('-t', '--threshold', type=float, default=0.5, help='network output required to be considered an activation')
    ap.add_argument('--calc-threshold', action='store_true', help="also print precise-calc-threshold's mu and std")
    ap.add_argument('-s', '--smoothing', type=float, default=1.2, help='extra smoothing of --calc-threshold')
    ap.add_argument('--device', type=int, default=0)
    args = ap.parse_args(argv)

    from .core import PreciseB200
    from .offline import TrainState, calc_threshold, test_pool, test_rows, vectorize_clips
    from .params import ListenerParams
    from .runner import _resolve_model
    from .simulate import check_pool_models, check_train_models
    models = [_resolve_model(m) for m in args.model]
    models = [(model, pr or ListenerParams()) for model, pr in models]
    wide = any(m.hidden > 24 for m, _ in models)
    (check_train_models if wide else check_pool_models)(args.model, models)
    model, pr = models[0]
    files, clips, targets = load_folder(args.folder, args.use_train, pr.sample_rate)
    core = PreciseB200(pr, hidden=model.hidden, device=args.device, activation=model.activation,
                       recurrent_activation=model.recurrent_activation)
    kw = dict(thresholds=(args.threshold,), misses=True, miss_threshold=args.threshold)
    if wide:
        inputs = vectorize_clips(core, clips)
        state = TrainState.from_models(core, [m for m, _ in models], [0] * len(models))
        stats, missed = test_rows(core, state, inputs, targets, **kw)
    else:
        core.set_pool(len(models))
        for i, (m, p) in enumerate(models):
            core.pool_load(i, m, p)
        stats, missed = test_pool(core, clips, targets, np.arange(len(models), dtype=np.int32), **kw)
    for name, st, miss in zip(args.model, stats, missed):
        print('=== %s ===' % name)
        if not args.no_filenames:
            print('=== False Positives ===')
            print('\n'.join(files[i] for i in miss if not targets[i]))
            print()
            print('=== False Negatives ===')
            print('\n'.join(files[i] for i in miss if targets[i]))
            print()
        print(st.counts_str(args.threshold))
        print()
        print(st.summary_str(args.threshold))
        if args.calc_threshold:
            fit = calc_threshold(st, args.smoothing)
            print('No data (or all NaN)' if fit is None else 'Peak: {:.2f} mu, {:.2f} std'.format(*fit))
    core.close()


if __name__ == '__main__':
    main()
