"""Times pb_train_wide (csrc/train_wide.cuh) against the torch baseline of scripts/train_time.py at the same hidden size, and
against pb_train at H = 20, on the same GPU.

    python scripts/train_wide_time.py [--out FILE.json] [--quick]

Workloads: H in {20, 32, 64, 128} x k in {1, 64, 256} networks x 5 000 entries per network (every network on the same
clips), batch sizes 256 and 5 000, the default front end (F = 13, T = 29), dropout 0.2, one epoch per timed call after a
warm-up epoch.  The baseline is train_time.py's torch_epoch (bmm over the rows, a Python loop over the steps, autograd,
RMSprop) at hidden size H.

Reported per workload: seconds per epoch, entry-steps per second (entries x epochs / s, train_time.py's unit) and FLOP/s.
FLOP per entry and epoch are train_time.py's count at H: T x 3 x (2 x 3H x F + 2 x 3H x H), the forward's products and the
backward's two per weight matrix, each counted once.  The kernel runs each product as three TF32 products (the 3xTF32
split), so it executes three times that count: "tc_frac" is 3 x the useful FLOP/s against the H100 SXM data sheet's
495 TFLOP/s dense TF32, the share of the tensor cores the kernel keeps busy.  The card's name, power limit and maximum SM
clock are read in the same run.  --quick: k = 1 and 64 only.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

import train_time  # noqa: E402

F, T = 13, 29
N = 5000
PEAK_TF32 = 495e12


def flop_per_entry(H):
    return T * 3 * (2 * 3 * H * F + 2 * 3 * H * H)


def rows_of(models, stride):
    w = np.zeros((len(models), stride), np.float32)
    for i, m in enumerate(models):
        flat = np.concatenate([m.kernel.ravel(), m.recurrent.ravel(), m.bias, m.dense_w, [0.0]])
        w[i, :flat.size] = flat
    return w


def time_device(torch, core, x, y, rows, w, bs):
    dw = torch.from_numpy(w).cuda()
    drms = torch.zeros_like(dw)
    core.train(x, y, rows, dw, drms, epochs=1, batch_size=bs)                  # warm-up
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    core.train(x, y, rows, dw, drms, epochs=1, epoch0=1, batch_size=bs)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3


def time_torch(torch, x, yt, models, H, bs):
    train_time.H = H                        # torch_epoch reads the module's hidden size
    k = len(models)
    K = torch.from_numpy(np.stack([m.kernel for m in models])).cuda()
    U = torch.from_numpy(np.stack([m.recurrent for m in models])).cuda()
    bb = torch.zeros(k, 3 * H, device='cuda')
    dwt = torch.from_numpy(np.stack([m.dense_w for m in models])).cuda()
    dbt = torch.zeros(k, device='cuda')
    state = [torch.zeros_like(p) for p in (K, U, bb, dwt, dbt)]
    train_time.torch_epoch(torch, x, yt, K, U, bb, dwt, dbt, state, bs)        # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    train_time.torch_epoch(torch, x, yt, K, U, bb, dwt, dbt, state, bs)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='also write the results as JSON to this file')
    ap.add_argument('--quick', action='store_true', help='k = 1 and 64 only')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('train_wide_time.py measures on a CUDA device; none found')
    from mycroft_precise_b200 import GruModel, PreciseB200
    from mycroft_precise_b200.core import PB_TRAIN_STRIDE, PB_TRAIN_WIDE_STRIDE
    info = train_time.card()
    core = PreciseB200()
    rs = np.random.RandomState(0)
    x = torch.from_numpy(rs.randn(N, T, F).astype(np.float32)).cuda()
    y = (rs.rand(N) < 0.3).astype(np.uint8)
    yt = torch.from_numpy(y.astype(np.float32)).cuda()
    results = []
    for H in (20, 32, 64, 128):
        for k in ((1, 64) if args.quick else (1, 64, 256)):
            models = [GruModel.init(F, H, i) for i in range(k)]
            rows = core.train_rows([H] * k, ['linear'] * k, ['hard_sigmoid'] * k, list(range(k)))
            for bs in (256, 5000):
                es = k * N
                r = dict(H=H, k=k, entries=N, batch_size=bs)
                r['wide_s'] = time_device(torch, core, x, y, rows, rows_of(models, PB_TRAIN_WIDE_STRIDE), bs)
                if H == 20:
                    r['pb_train_s'] = time_device(torch, core, x, y, rows, rows_of(models, PB_TRAIN_STRIDE), bs)
                    r['pb_train_entry_steps_per_s'] = es / r['pb_train_s']
                r['torch_s'] = time_torch(torch, x, yt, models, H, bs)
                fl = es * flop_per_entry(H)
                r.update(wide_entry_steps_per_s=es / r['wide_s'], torch_entry_steps_per_s=es / r['torch_s'],
                         speedup_vs_torch=r['torch_s'] / r['wide_s'], wide_tflops=fl / r['wide_s'] / 1e12,
                         torch_tflops=fl / r['torch_s'] / 1e12, tc_frac=3 * fl / r['wide_s'] / PEAK_TF32)
                results.append(r)
                print(json.dumps(r), flush=True)
    core.close()
    out = dict(card=info, flop_per_entry={H: flop_per_entry(H) for H in (20, 32, 64, 128)}, peak_tf32=PEAK_TF32,
               results=results)
    print('card:', info)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
