"""Times generated training audio (pb_generate, csrc/generate.cuh; offline.Generator, train_generated) on the GPU.

    python scripts/generated_time.py [--out FILE.json]

Workload: precise-train-generated's default epoch, 100 steps x 200 windows = 20 000 windows at chunk 2 048 and the default
front end, over 32 seeded backgrounds of 30 .. 120 s and 40 wake-word / 40 not-wake-word clips of 0.75 .. 1.25 s; and the
same at 10x the windows.  For each: the host plan (Generator.plan + tables), pb_generate with d_inputs (CUDA events around
Generator.run), and one pb_train epoch of one H = 20 network at batch 200 (CUDA events).  For comparison, the literal form
(oracle/generated.py, the reference's per-chunk loop with the oracle Listener's MFCC) on the CPU over 200 chunks, per chunk.
Each device number is the median of several repetitions after a warm-up.  The card's name, power limit and maximum SM
clock are read in the same run.
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


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                                      # noqa: BLE001
        return 'unknown (%s)' % e


def events(torch, fn, reps):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return float(np.median(out))


def data():
    rs = np.random.RandomState(0)
    sig = lambda n, a: np.clip(np.round(rs.randn(int(n)) * a), -32768, 32767).astype(np.int16)
    bgs = [sig(n, 300 + 50 * i) for i, n in enumerate(rs.randint(30 * 16000, 120 * 16000, 32))]
    wake = [sig(n, 3000) for n in rs.randint(12000, 20000, 40)]
    other = [sig(n, 2000) for n in rs.randint(12000, 20000, 40)]
    return bgs, wake, other


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='also write the results as JSON here')
    args = ap.parse_args()
    import torch
    import mycroft_precise_b200 as m
    from mycroft_precise_b200.offline import Generator, TrainState
    from oracle import generated as og
    from oracle.listener import OracleListener
    from oracle.params import OracleParams
    core = m.PreciseB200()
    bgs, wake, other = data()
    res = {'card': card()}
    state = TrainState.from_models(core, [m.GruModel.init(13, 20, 0)], [0])
    for name, n in (('default', 20000), ('x10', 200000)):
        gen = Generator(core, bgs, wake, other, chunk=2048, seed=1)
        t = time.perf_counter()
        plan = gen.plan(n)
        gen.tables(plan)
        plan_ms = 1e3 * (time.perf_counter() - t)
        box = {}
        gen_ms = events(torch, lambda: box.update(r=gen.run(plan)), 5)
        x, tg = box['r'][0], box['r'][1]
        train_ms = events(torch, lambda: core.train(x, tg, state.rows, state.weights, state.rms, epochs=1, batch_size=200), 5)
        items, _, _, _ = gen.tables(plan)
        res[name] = dict(windows=n, items=len(plan), samples=int(items['length'].sum()), positives=float(tg.mean()),
                         plan_ms=plan_ms, generate_ms=gen_ms, train_ms=train_ms)
        print(name, res[name], flush=True)
    gen = Generator(None, bgs, wake, other, chunk=2048, seed=1, sample_rate=16000, buffer_samples=24000)
    lit = og.Literal(wake, other, lambda kind, k: 0.3 if kind != 'piece' else (0.7 if k % 4 == 0 else 0.3), 2048, 16000, 24000)
    lis = OracleListener(None, OracleParams(), 2048)
    t = time.perf_counter()
    merged, _ = lit.file(bgs[0][:201 * 2048])
    for c in merged:
        lis.update_vectors(c)
    res['literal_cpu_ms_per_chunk'] = 1e3 * (time.perf_counter() - t) / merged.shape[0]
    print('literal', res['literal_cpu_ms_per_chunk'], 'ms per chunk')
    core.close()
    print(json.dumps(res))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
