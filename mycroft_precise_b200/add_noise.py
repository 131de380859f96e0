"""``precise-add-noise`` on the GPU (reference: precise/scripts/add_noise.py): a copy of a dataset with background noise
mixed into every clip.

    python -m mycroft_precise_b200.add_noise FOLDER NOISE_FOLDER OUTPUT_FOLDER [-if N] [-nl LOW] [-nh HIGH] [--seed S]
                                             [--device D]

The clips are FOLDER's wake-word, not-wake-word, test/wake-word and test/not-wake-word wavs, in that order (the reference's
train_files + test_files), sorted by path within each group.  The noise is NOISE_FOLDER/*.wav (not recursive, sorted), read
as one cyclic stream whose position carries over from clip to clip and copy to copy.  Each clip gets N noisy copies, written
as x.wav (copy 0) and x.<n>.wav under the clip's relative directory in OUTPUT_FOLDER, 16-bit mono at the default
ListenerParams' sample rate.  Copy n of a clip mixes at ratio LOW + (HIGH - LOW) u, u the next random.Random(S).random() in
processing order: the sequence the reference draws after random.seed(S).  The mix is pb_add_noise's (include/precise_b200.h):
a silent noise span adds no noise and out-of-range values saturate, where the reference gives NaN and wraps.  Tags files
(the reference's -tg) are not read.
"""
import argparse
import glob
import os
import random
import wave
from os.path import join

import numpy as np

REPEAT_WARNING = 'Warning: Repeating noise 100+ times. Add more to prevent overfitting.'


def find_clips(folder: str):
    """The clips precise-add-noise processes, in its group order, sorted within each group."""
    from .test import find_wavs
    groups = list(find_wavs(folder)) + list(find_wavs(join(folder, 'test')))
    return [f for g in groups for f in sorted(g)]


def output_name(folder: str, source: str, n: int, output_folder: str) -> str:
    """translate_filename (add_noise.py:103-109): x.wav for copy 0, x.<n>.wav for copy n > 0."""
    relative = os.path.relpath(os.path.abspath(source), os.path.abspath(folder))
    if n > 0:
        base, ext = os.path.splitext(relative)
        relative = base + '.' + str(n) + ext
    return join(output_folder, relative)


def write_wav(path: str, pcm: np.ndarray, sample_rate: int):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with wave.open(path, 'wb') as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(sample_rate)
        w.writeframes(np.ascontiguousarray(pcm, '<i2').tobytes())


def main(argv=None):
    ap = argparse.ArgumentParser(prog='precise-add-noise', description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('folder', help='folder containing the source dataset')
    ap.add_argument('noise_folder', help='folder with wav files containing noise to be added')
    ap.add_argument('output_folder', help='folder to write the duplicate generated dataset')
    ap.add_argument('-if', '--inflation-factor', type=int, default=1, help='noisy samples generated per source sample')
    ap.add_argument('-nl', '--noise-ratio-low', type=float, default=0.0, help='minimum random ratio of noise to sample')
    ap.add_argument('-nh', '--noise-ratio-high', type=float, default=0.4, help='maximum random ratio of noise to sample')
    ap.add_argument('--seed', type=int, default=None, help='seed of the ratios (default: unseeded)')
    ap.add_argument('--device', type=int, default=0)
    args = ap.parse_args(argv)

    from .core import PreciseB200
    from .offline import NoiseSource, add_noise
    from .params import ListenerParams
    from .simulate import read_wav
    pr = ListenerParams()
    files = find_clips(args.folder)
    noise = [read_wav(f, pr.sample_rate) for f in sorted(glob.glob(join(args.noise_folder, '*.wav')))]
    if sum(n.shape[0] for n in noise) == 0:
        raise SystemExit('no noise audio in %s/*.wav: nothing to mix' % args.noise_folder)
    clips = [read_wav(f, pr.sample_rate) for f in files]
    M = int(args.inflation_factor)
    rnd = random.Random(args.seed)
    lo, hi = args.noise_ratio_low, args.noise_ratio_high
    ratios = np.asarray([lo + (hi - lo) * rnd.random() for _ in range(len(files) * M)], np.float64)
    items = np.repeat(np.arange(len(files)), M)

    core = PreciseB200(pr, device=args.device)
    source = NoiseSource(core, noise)
    out, offsets = add_noise(core, clips, source, ratios, items)
    out = out.cpu().numpy()
    core.close()
    N = len(source)
    for p, (i, n) in enumerate(zip(items.tolist(), [n for _ in files for n in range(M)])):
        write_wav(output_name(args.folder, files[i], n, args.output_folder), out[offsets[p]:offsets[p + 1]], pr.sample_rate)
        if offsets[p + 1] // N >= 100 > offsets[p] // N:                  # the corpus has been read through 100 times
            print(REPEAT_WARNING)
    print('Done!')
    return out, offsets


if __name__ == '__main__':
    main()
