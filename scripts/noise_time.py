"""Times noise augmentation (pb_add_noise, csrc/noise.cuh) on the GPU.

    python scripts/noise_time.py [--out FILE.json]

Workloads, all at the default front end (F = 13, T = 29, max_samples 24 000), with seeded int16 clips and an int16 noise
corpus of one hour (57.6 M samples):
  mix      pb_add_noise with d_out only over 4 096 clips of 16 000 .. 48 000 samples (about 131 M samples).  Its bytes are
           what the algorithm must move: the clip and its noise span read twice (the sums pass and the mix pass) and the
           output written once, 2 x (2 + 2) + 2 = 10 bytes per sample; over the measured time, against the H100 SXM's
           3.35 TB/s.
  vector   offline.vectorize_noisy against offline.vectorize_clips on the same 4 096 clips, end to end, and pb_add_noise
           (d_inputs only) against pb_vectorize_clips on the clips already packed on the device: what mixing adds to K1.
  epoch    one offline.train epoch of one H = 20 network on 2 048 clips, with Augment(copies = 1) and without.
Each is warmed up, then timed with CUDA events over several repetitions (median reported).  The card's name, power limit
and maximum SM clock are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM = 3.35e12


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                                      # noqa: BLE001
        return 'unknown (%s)' % e


def timed(torch, fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e-3)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    import mycroft_precise_b200 as m
    assert torch.cuda.is_available(), 'noise_time needs a GPU'
    rs = np.random.RandomState(0)
    core = m.PreciseB200()
    n = 4096
    clips = [np.clip(rs.randn(int(L)) * 2000, -32768, 32767).astype(np.int16) for L in rs.randint(16000, 48001, n)]
    noise = np.clip(rs.randn(3600 * 16000) * 1500, -32768, 32767).astype(np.int16)
    ratios = rs.rand(n) * 0.4
    res = dict(card=card())

    # mix: one library call over packed clips
    pcm, offsets, entry = m.offline._pack(core, clips)
    dnoise = torch.from_numpy(noise).cuda()
    items = entry.astype(np.int32)
    samples = int(sum(c.shape[0] for c in clips))
    t = timed(torch, lambda: core.add_noise(pcm, offsets, dnoise, items, ratios, 12345), 20)
    nbytes = 10 * samples
    res['mix'] = dict(clips=n, samples=samples, seconds=t, bytes=nbytes, bytes_per_s=nbytes / t, hbm_frac=nbytes / t / HBM)

    # vectorize_noisy against vectorize_clips, end to end (host clips packed per call) and as library calls on clips already
    # on the device (lengths rounded down to multiples of 8, so both take the fast K1 on every clip)
    src = m.offline.NoiseSource(core, [noise])
    tv = timed(torch, lambda: m.offline.vectorize_noisy(core, clips, src, ratios), 10)
    tc = timed(torch, lambda: m.offline.vectorize_clips(core, clips), 10)
    c8 = [c[:c.shape[0] // 8 * 8] for c in clips]
    pcm8, off8, entry8 = m.offline._pack(core, c8)
    lv = timed(torch, lambda: core.add_noise(pcm8, off8, dnoise, entry8.astype(np.int32), ratios, 12345, out=False, inputs=True), 20)
    lc = timed(torch, lambda: core.vectorize_clips(pcm8, off8), 20)
    res['vector'] = dict(clips=n, noisy_seconds=tv, clean_seconds=tc, library_noisy_seconds=lv, library_clean_seconds=lc,
                         library_added_seconds=lv - lc)

    # one augmented epoch against one plain epoch
    k = 2048
    tg = (np.arange(k) % 2).astype(np.uint8)
    init = m.GruModel.init(13, 20, 0)
    inputs = m.offline.vectorize_clips(core, clips[:k])
    state = m.offline.TrainState.from_models(core, [init], [0])
    tp = timed(torch, lambda: m.offline.train(core, state, inputs, tg, epochs=1), 5)
    aug = m.offline.Augment(src, 1, 0.0, 0.4, 0)
    ta = timed(torch, lambda: m.offline.train(core, state, clips[:k], tg, epochs=1, augment=aug), 5)
    res['epoch'] = dict(clips=k, plain_seconds=tp, augmented_seconds=ta)
    core.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
