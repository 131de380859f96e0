"""Model bank vs independent handles at the bench size (DESIGN.md §3 "K2 for a model bank", §6).

131 072 streams, M in {1, 2, 4} default-shaped networks (H = 20 over 13 MFCCs) with seeded weights and seeded PCM.
  arm a: one handle holding the M models (StreamBatch.add_model), one update_models per tick;
  arm b: M one-model StreamBatches, one update each per tick.
The arms alternate in one process (REPS rounds).  Each round primes PRIME untimed ticks, then times TIMED ticks: K1 / K2 from the
library's CUDA-event profile (pb_profile_*, slots 0 / 1, summed over an arm's handles), tick time from CUDA events around the
timed loop.  Both arms see the same tick sequence, so their last-tick raw outputs must agree per model within 1e-5.

    python scripts/bank_time.py [--models 1 2 4] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np                      # noqa: E402
import torch                            # noqa: E402
import mycroft_precise_b200 as m        # noqa: E402

S, PRIME, TIMED, REPS = 131072, 30, 20, 2


def card():
    """Name, power limit and max SM clock of cuda:0, read in the same run as the timings."""
    try:
        q = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ''
    return q or torch.cuda.get_device_name(0) + ' (power limit not readable)'


def timed(handles, tick, pcm):
    for i in range(PRIME):
        tick(pcm[i & 1])
    torch.cuda.synchronize()
    for h in handles:
        h.core.profile(True)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for i in range(TIMED):
        out = tick(pcm[i & 1])
    t1.record()
    torch.cuda.synchronize()
    k1 = k2 = 0.0
    for h in handles:
        ms, _ = h.core.profile_read()
        k1 += ms[0]
        k2 += ms[1]
        h.core.profile(False)
    us = 1e3 / TIMED
    return dict(k1_us=k1 * us, k2_us=k2 * us, tick_us=t0.elapsed_time(t1) * us), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--models', type=int, nargs='+', default=[1, 2, 4])
    ap.add_argument('--out', default=None, help='also write the results as JSON to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bank_time.py needs a CUDA device')
    gpu = card()
    print('card:', gpu, flush=True)
    models = [m.GruModel.random(13, 20, seed=i, scale=0.1) for i in range(max(args.models))]
    pcm = [torch.from_numpy(np.clip(np.random.RandomState(i).randn(S, 1024) * 3000, -32768, 32767).astype(np.int16)).cuda()
           for i in range(2)]
    results = []
    for M in args.models:
        bank = m.StreamBatch(models[0], S)
        for mod in models[1:M]:
            bank.add_model(mod)
        solo = [m.StreamBatch(mod, S) for mod in models[:M]]
        for rep in range(REPS):
            ta, oa = timed([bank], bank.update_models, pcm)
            tb, ob = timed(solo, lambda p: [sb.update(p)['raw'] for sb in solo], pcm)
            err = max(float((oa['raw'][i] - ob[i]).abs().max()) for i in range(M))
            print('M=%d round %d  a (bank, update_models): K1 %.1f us  K2 %.1f us  tick %.1f us | b (%d handles, update): '
                  'K1 %.1f us  K2 %.1f us  tick %.1f us | max |raw a - raw b| %.3g'
                  % (M, rep, ta['k1_us'], ta['k2_us'], ta['tick_us'], M, tb['k1_us'], tb['k2_us'], tb['tick_us'], err), flush=True)
            assert err < 1e-5, err
            results.append(dict(models=M, round=rep, a=ta, b=tb, max_raw_diff=err))
        bank.core.close()
        for sb in solo:
            sb.core.close()
        del bank, solo
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(dict(card=gpu, streams=S, prime=PRIME, timed=TIMED, results=results), f, indent=1)


if __name__ == '__main__':
    main()
