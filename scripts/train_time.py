"""Times pb_train (csrc/train.cuh) against the same math in torch on the same GPU.

    python scripts/train_time.py [--out FILE.json] [--quick]

Workloads: k in {1, 64, 1024} networks x {500, 5000} entries per network (every network on the same clips, the
train-optimize case), batch sizes 256 and 5000, H = 20 at the default front end (F = 13, T = 29), dropout 0.2, one epoch
per timed call.  The baseline is what a torch user would write: per batch, the rows' weights as batched tensors (bmm over
the rows, in chunks of rows that fit in memory), a Python loop over the 29 steps, autograd, and RMSprop with Keras's
epsilon placement (w -= lr g / (sqrt(a) + eps)); its shuffles and masks come from torch's generator.

Reported per workload: seconds per epoch for both, entry-steps per second (entries x epochs / s) and the kernel's FP32
FLOP/s against the H100 SXM data sheet's 67 TFLOP/s.  FLOP per entry and epoch are counted from the shapes:
T x 3 x (2 x 3H x F + 2 x 3H x H) -- the forward's input and recurrent products and the backward's two products per
weight matrix (input and weight gradients); activations and the Dense layer are left out.  The card's name, power limit
and maximum SM clock are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H, F, T = 20, 13, 29
PEAK_FP32 = 67e12


def flop_per_entry():
    return T * 3 * (2 * 3 * H * F + 2 * 3 * H * H)


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:                                      # noqa: BLE001
        return 'unknown (%s)' % e


def torch_epoch(torch, x, y, K, U, b, dw, db, state, bs, rate=0.2, lr=1e-3, rho=0.9, eps=1e-7, bias=0.8, chunk_entries=1 << 19):
    """One epoch of the baseline over rows [k] sharing inputs x [n, T, F]."""
    k, n = K.shape[0], x.shape[0]
    perm = torch.argsort(torch.rand(k, n, device=x.device), 1)
    params = [K, U, b, dw, db]
    for b0 in range(0, n, bs):
        B = min(bs, n - b0)
        idx = perm[:, b0:b0 + B]
        rc = max(1, chunk_entries // B)
        grads = [torch.zeros_like(p) for p in params]
        for r0 in range(0, k, rc):
            r1 = min(k, r0 + rc)
            ps = [p[r0:r1].detach().requires_grad_(True) for p in params]
            Kc, Uc, bc, dwc, dbc = ps
            xb = x[idx[r0:r1]]                                   # [kc, B, T, F]
            yb = y[idx[r0:r1]]
            m = (torch.rand(r1 - r0, B, 3, F, device=x.device) >= rate).float() / (1 - rate)
            h = torch.zeros(r1 - r0, B, H, device=x.device)
            for t in range(T):
                xt = xb[:, :, t, :]
                az = torch.bmm(xt * m[:, :, 0], Kc[:, :, :H]) + bc[:, None, :H] + torch.bmm(h, Uc[:, :, :H])
                ar = torch.bmm(xt * m[:, :, 1], Kc[:, :, H:2 * H]) + bc[:, None, H:2 * H] + torch.bmm(h, Uc[:, :, H:2 * H])
                z = torch.clamp(0.2 * az + 0.5, 0, 1)
                r = torch.clamp(0.2 * ar + 0.5, 0, 1)
                hh = torch.bmm(xt * m[:, :, 2], Kc[:, :, 2 * H:]) + bc[:, None, 2 * H:] + torch.bmm(r * h, Uc[:, :, 2 * H:])
                h = z * h + (1 - z) * hh
            p = torch.sigmoid(torch.bmm(h, dwc[:, :, None])[..., 0] + dbc[:, None])
            loss = (bias * (-(1 - yb) * torch.log(1 - p + 1e-7)) + (1 - bias) * (-yb * torch.log(p + 1e-7))).sum() / B
            gs = torch.autograd.grad(loss, ps)
            for g, gc in zip(grads, gs):
                g[r0:r1] = gc
        with torch.no_grad():
            for p, g, a in zip(params, grads, state):
                a.mul_(rho).addcmul_(g, g, value=1 - rho)
                p.sub_(lr * g / (a.sqrt() + eps))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='also write the results as JSON to this file')
    ap.add_argument('--quick', action='store_true', help='k = 1 and 64 only')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('train_time.py measures on a CUDA device; none found')
    from mycroft_precise_b200 import GruModel, PreciseB200
    from mycroft_precise_b200.core import PB_TRAIN_STRIDE
    info = card()
    core = PreciseB200()
    rs = np.random.RandomState(0)
    results = []
    ev = lambda: torch.cuda.Event(enable_timing=True)
    for k in ((1, 64) if args.quick else (1, 64, 1024)):
        for n in (500, 5000):
            x = torch.from_numpy(rs.randn(n, T, F).astype(np.float32)).cuda()
            y = (rs.rand(n) < 0.3).astype(np.uint8)
            yt = torch.from_numpy(y.astype(np.float32)).cuda()
            models = [GruModel.init(F, H, i) for i in range(k)]
            w = np.zeros((k, PB_TRAIN_STRIDE), np.float32)
            for i, m in enumerate(models):
                flat = np.concatenate([m.kernel.ravel(), m.recurrent.ravel(), m.bias, m.dense_w, [0.0]])
                w[i, :flat.size] = flat
            rows = core.train_rows([H] * k, ['linear'] * k, ['hard_sigmoid'] * k, list(range(k)))
            for bs in (256, 5000):
                dw = torch.from_numpy(w).cuda()
                drms = torch.zeros_like(dw)
                core.train(x, y, rows, dw, drms, epochs=1, batch_size=bs)           # warm-up
                torch.cuda.synchronize()
                reps = 3 if k * n <= 64 * 5000 else 1
                a, b = ev(), ev()
                a.record()
                for e in range(reps):
                    core.train(x, y, rows, dw, drms, epochs=1, epoch0=1 + e, batch_size=bs)
                b.record()
                torch.cuda.synchronize()
                t_kernel = a.elapsed_time(b) / 1e3 / reps
                # torch baseline
                K = torch.from_numpy(np.stack([m.kernel for m in models])).cuda()
                U = torch.from_numpy(np.stack([m.recurrent for m in models])).cuda()
                bb = torch.zeros(k, 3 * H, device='cuda')
                dwt = torch.from_numpy(np.stack([m.dense_w for m in models])).cuda()
                dbt = torch.zeros(k, device='cuda')
                state = [torch.zeros_like(p) for p in (K, U, bb, dwt, dbt)]
                torch_epoch(torch, x, yt, K, U, bb, dwt, dbt, state, bs)         # warm-up
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                torch_epoch(torch, x, yt, K, U, bb, dwt, dbt, state, bs)
                torch.cuda.synchronize()
                t_torch = time.perf_counter() - t0
                es = k * n
                r = dict(k=k, entries=n, batch_size=bs, kernel_s=t_kernel, torch_s=t_torch,
                         kernel_entry_steps_per_s=es / t_kernel, torch_entry_steps_per_s=es / t_torch,
                         speedup=t_torch / t_kernel, kernel_tflops=es * flop_per_entry() / t_kernel / 1e12,
                         kernel_frac_fp32_peak=es * flop_per_entry() / t_kernel / PEAK_FP32)
                results.append(r)
                print(json.dumps(r), flush=True)
    core.close()
    out = dict(card=info, flop_per_entry=flop_per_entry(), peak_fp32=PEAK_FP32, results=results)
    print('card:', info)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
