"""Recorded corpora at scale (DESIGN.md §3 "Recorded corpora", §6).

A seeded synthetic corpus generated on the device: recordings of 5 s to 20 min (5 s x 240^(u^1.3), u uniform: about 2 000
of them in 100 h), HOURS hours in all, int16 noise
with the bench's edge streams (silence, full scale) among them, packed at 8-sample-aligned offsets.  A default-shaped
network (H = 20 over 13 MFCCs) with seeded weights.
  listener, c = 1024: pb_score_corpus, then the A arm: one StreamBatch-style ragged tick per chunk over every recording
                      still running (update_ragged), raw compared;
  simulate, c = 4096: pb_score_corpus, then the A arm: offline.evaluate per recording plus a host TriggerDetector,
                      raw, activations and activated chunks compared.
Reported: hours of audio per second of device time (CUDA events around the call), per-kernel times from the library's
CUDA-event profile (slot 0: MFCC with its plan, slot 1: network and trigger), K1 bytes per second against the byte model
(PCM read once, 2 B per sample, plus the frame rows written, row_stride * 4 B per row; the fast K1 actually fetches 512 of
every 800 samples, 1 KB per frame, which k1_fetched_GBps reports), K2 windows per second, and the
per-recording trigger pass of one one-hour recording (slot 1 with the trigger outputs minus slot 1 without them).

    python scripts/corpus_time.py [--hours 100] [--out result.json]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np                      # noqa: E402
import torch                            # noqa: E402
import mycroft_precise_b200 as m        # noqa: E402
from mycroft_precise_b200 import offline   # noqa: E402
from mycroft_precise_b200.core import _ptr  # noqa: E402
from mycroft_precise_b200.runner import TriggerDetector   # noqa: E402
from bank_time import card              # noqa: E402

SR = 16000


def corpus(hours, seed=0):
    rs = np.random.RandomState(seed)
    lens = []
    while sum(lens) < hours * 3600 * SR:
        lens.append(int(5 * 240 ** (rs.uniform() ** 1.3) * SR) & ~7)    # 5 s .. 20 min, mean about 178 s
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    g = torch.Generator(device='cuda').manual_seed(seed)
    pcm = torch.empty(int(offs[-1]), dtype=torch.int16, device='cuda')
    step = 1 << 28
    for a in range(0, pcm.numel(), step):
        n = min(step, pcm.numel() - a)
        pcm[a:a + n] = (torch.randn(n, generator=g, device='cuda') * 3000).clamp_(-32768, 32767).to(torch.int16)
    pcm[offs[1]:offs[2]] = 0                               # edge streams: silence and full scale
    pcm[offs[2]:offs[3]] = 32767
    return pcm, offs


def timed_call(core, *args):
    core.profile(True)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    out = core.score_corpus(*args)
    t1.record()
    torch.cuda.synchronize()
    ms, _ = core.profile_read()
    core.profile(False)
    return out, t0.elapsed_time(t1), ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--hours', type=float, default=100.0)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    res = dict(card=card(), hours=args.hours)
    model = m.GruModel.random(13, 20, seed=0, scale=0.1)
    core = m.PreciseB200()
    core.load_weights(model.kernel, model.recurrent, model.bias, model.dense_w, model.dense_b)
    pcm, offs = corpus(args.hours)
    n_rec, n_samp = len(offs) - 1, int(offs[-1])
    nf = sum(core.mfcc_frames(int(L)) for L in np.diff(offs))
    rows = 1 + nf + n_rec * (core.n_features - 1)
    k1_bytes = 2 * n_samp + rows * 16 * 4
    k1_fetched = 1024 * nf + rows * 16 * 4
    res.update(recordings=n_rec, samples=n_samp, frames=nf, k1_model_bytes=k1_bytes, k1_fetched_bytes=k1_fetched)
    hours = n_samp / SR / 3600
    lens = np.diff(offs)
    for sched, c in (('listener', 1024), ('simulate', 4096)):
        core.score_corpus(pcm, offs, sched, c)                # warm-up
        torch.cuda.synchronize()
        out, ms, prof = timed_call(core, pcm, offs, sched, c, 0.5)
        W = out['raw'].shape[1]
        r = dict(windows=W, call_ms=ms, k1_ms=prof[0], k2_trigger_ms=prof[1],
                 hours_per_device_s=hours / (ms / 1e3), k1_GBps=k1_bytes / (prof[0] / 1e3) / 1e9,
                 k1_fetched_GBps=k1_fetched / (prof[0] / 1e3) / 1e9,
                 windows_per_s=W / (prof[1] / 1e3))
        wo = np.concatenate([[0], np.cumsum([core.corpus_windows(int(L), sched, c) for L in lens])])
        raw = out['raw'][0]
        t0 = time.perf_counter()
        if sched == 'simulate':
            errs, act_ok, above_ok = 0.0, 0, 0
            acts = out['activations'][0].cpu().numpy()
            above = out['above'][0].cpu().numpy()
            for i in range(n_rec):
                p = offline.evaluate(core, pcm[offs[i]:offs[i + 1]], c)
                if p.numel():
                    errs = max(errs, float((p - raw[wo[i]:wo[i + 1]]).abs().max()))
                ph = p.cpu().numpy()
                det = TriggerDetector(c, trigger_level=0, sensitivity=0.5)
                act_ok += int(sum(det.update(x) for x in ph) == acts[i])
                above_ok += int((ph > 0.5).sum() == above[i])
            torch.cuda.synchronize()
            r.update(a_arm_s=time.perf_counter() - t0, a_arm_max_raw_err=errs, a_arm_activations_equal=act_ok,
                     a_arm_above_equal=above_ok)
        else:
            starts = torch.from_numpy(offs[:-1]).cuda()
            K = torch.from_numpy(lens // c).cuda()
            sb = m.StreamBatch(model, n_rec, chunk_samples=c)
            ar = torch.arange(c, device='cuda')
            tick_raw = torch.full((n_rec, int(K.max())), float('nan'), device='cuda')
            for k in range(int(K.max())):
                act = torch.nonzero(K > k)[:, 0]
                chunk = pcm[(starts[act, None] + k * c + ar).reshape(-1)]
                o = sb.update_ragged(chunk, torch.arange(act.numel() + 1, device='cuda') * c, act.to(torch.int32), c)
                tick_raw[act, k] = o['raw'][0]
            torch.cuda.synchronize()
            r['a_arm_s'] = time.perf_counter() - t0
            Kh = lens // c
            mask = torch.arange(tick_raw.shape[1], device='cuda')[None, :] < K[:, None]
            r['a_arm_max_raw_err'] = float((tick_raw[mask] - raw).abs().max())
            assert tick_raw[mask].numel() == W == int(Kh.sum())
        res[sched] = r
        print(sched, json.dumps(r), flush=True)
    # the trigger pass over one one-hour recording: slot 1 with the trigger outputs minus slot 1 with raw only
    one = pcm[:3600 * SR].contiguous()
    o1 = np.array([0, one.numel()], np.int64)
    W = core.corpus_windows(one.numel(), 'listener', 1024)
    rawb = torch.empty(W, device='cuda')
    t_raw, t_all = [], []
    for _ in range(3):
        core.profile(True)
        core.lib.pb_score_corpus(core._h, _ptr(one), o1.ctypes.data_as(C.c_void_p), 1, 32768, 0, 1024, 0.5, _ptr(rawb),
                                 None, None, None, None, None, core._stream())
        torch.cuda.synchronize()
        t_raw.append(core.profile_read()[0][1])
        _, _, prof = timed_call(core, one, o1, 'listener', 1024, 0.5)
        t_all.append(prof[1])
    res['trigger_one_hour_ms'] = float(np.median(t_all) - np.median(t_raw))
    res['one_hour_windows'] = W
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
