"""K1 of the default tick: the pipelined FFT kernel (k1 mode 0) against the kernel it replaced (k1 mode 2), DESIGN.md §3, §6.

131 072 streams, the default network (H = 20 over 13 MFCCs) with seeded weights, seeded PCM, one `update` per tick.  Each arm is a
(library, k1 mode) pair run in a subprocess of its own; the arms alternate, ROUNDS rounds each.  A round primes PRIME untimed
ticks, then times TIMED ticks with the library's CUDA-event profile (pb_profile_*, slot 0 = K1, slot 1 = K2).  Every round sees
the same tick sequence, so the last tick's raw / conf / fired and the streams' exported state (ring, tail, n_samples) must be
bit-identical across all arms and rounds.

Bytes per tick come from the streams' sample counts, which all streams share here (every stream takes the same 1024-sample
chunk on every tick): per stream, the 1 KB input of every frame the tick completes (read from the old tail and the chunk), the
part of the old tail a short chunk shifts (read + written), the chunk samples that become the new tail (read + written), the
MFCC rows (n_out floats each) and the sample counter (read + written).  Achieved TB/s is that over the K1 time, against the
H100 SXM data sheet's 3.35 TB/s of HBM3.

    python scripts/k1_time.py [--arm NAME=LIB:MODE ...] [--rounds 3] [--out result.json]
(LIB 'tree' = this tree's library.)
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TREE_LIB = os.path.join(ROOT, 'mycroft_precise_b200', 'csrc', 'libprecise_b200.so')
S, PRIME, TIMED, CHUNK = 131072, 30, 50, 1024
HBM_BPS = 3.35e12
DEFAULT_ARMS = ['fft=tree:2', 'pipelined=tree:0']


def card():
    """Name, power limit, SM clock now and max SM clock of cuda:0, read in the same run as the timings."""
    try:
        q = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                            '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ''
    return q or 'power limit not readable'


def frames_ready(n, used, hop):
    return (n - used) // hop + 1 if n >= used else 0


def tick_bytes(n0, chunk, used, hop, n_out):
    """K1's bytes for one stream whose sample count goes from n0 to n0 + chunk."""
    n1 = n0 + chunk
    c0, c1 = frames_ready(n0, used, hop), frames_ready(n1, used, hop)
    ts1 = min(c1 * hop, n1)
    n_old = max(0, n0 - ts1)                   # old-tail samples the new tail keeps (chunk < 512)
    m = n1 - max(ts1, n0)                      # chunk samples that go to the tail
    return (c1 - c0) * 2 * used + 2 * 2 * n_old + 2 * 2 * m + (c1 - c0) * 4 * n_out + 2 * 8


def child(dump, mode):
    """One round on the library PRECISE_B200_LIB names, in k1 mode `mode`: prints one JSON line, writes the last tick's outputs
    and the exported stream state under dump."""
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    import mycroft_precise_b200 as m
    if not torch.cuda.is_available():
        sys.exit('k1_time.py needs a CUDA device')
    sb = m.StreamBatch(m.GruModel.random(13, 20, seed=0, scale=0.1), S, chunk_samples=CHUNK)
    sb.core.k1_mode(mode)
    p = sb.core.params
    used, hop, n_out = min(p.n_fft, p.window_samples), p.hop_samples, 13
    pcm = [torch.from_numpy(np.clip(np.random.RandomState(i).randn(S, CHUNK) * 3000, -32768, 32767).astype(np.int16)).cuda()
           for i in range(2)]
    for i in range(PRIME):
        sb.update(pcm[i & 1])
    torch.cuda.synchronize()
    sb.core.profile(True)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for i in range(TIMED):
        out = sb.update(pcm[(PRIME + i) & 1])
    t1.record()
    torch.cuda.synchronize()
    ms, launches = sb.core.profile_read()
    for k in ('raw', 'conf', 'fired'):
        np.save(os.path.join(dump, k + '.npy'), out[k].cpu().numpy())
    np.save(os.path.join(dump, 'state.npy'), sb.export_streams()['state'].cpu().numpy())
    nbytes = S * sum(tick_bytes((PRIME + i) * CHUNK, CHUNK, used, hop, n_out) for i in range(TIMED)) / TIMED
    us = 1e3 / TIMED
    print(json.dumps(dict(k1_us=ms[0] * us, k2_us=ms[1] * us, tick_us=t0.elapsed_time(t1) * us, k1_launches=launches[0],
                          k1_bytes_per_tick=nbytes, lib=sb.core.lib.pb_build_info().decode(),
                          gpu=torch.cuda.get_device_name(0))), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--arm', action='append', default=None, help="NAME=LIB:MODE, LIB a libprecise_b200.so or 'tree' (repeatable)")
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None, help='also write the results as JSON to this file')
    ap.add_argument('--child', default=None, help=argparse.SUPPRESS)
    ap.add_argument('--mode', type=int, default=0, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args.child, args.mode)
    arms = []
    for a in args.arm or DEFAULT_ARMS:
        name, rest = a.split('=', 1)
        lib, mode = rest.rsplit(':', 1)
        lib = TREE_LIB if lib == 'tree' else os.path.abspath(lib)
        if not os.path.isfile(lib):
            sys.exit('arm %s: %s is missing' % (name, lib))
        arms.append((name, lib, int(mode)))
    gpu = card()
    print('card (name, power limit, SM clock, max SM clock):', gpu, flush=True)
    import numpy as np
    results, ref = [], None
    for rnd in range(args.rounds):
        for name, lib, mode in arms:
            with tempfile.TemporaryDirectory() as dump:
                p = subprocess.run([sys.executable, os.path.abspath(__file__), '--child', dump, '--mode', str(mode)],
                                   env=dict(os.environ, PRECISE_B200_LIB=lib), capture_output=True, text=True)
                if p.returncode != 0:
                    sys.exit('arm %s round %d failed:\n%s%s' % (name, rnd, p.stdout, p.stderr))
                r = json.loads(p.stdout.strip().splitlines()[-1])
                outs = {k: np.load(os.path.join(dump, k + '.npy')) for k in ('raw', 'conf', 'fired', 'state')}
            if ref is None:
                ref = outs
            same = all(np.array_equal(outs[k].view(np.uint8), ref[k].view(np.uint8)) for k in outs)
            sec = r['k1_us'] * 1e-6
            r.update(arm=name, mode=mode, round=rnd, outputs_match_first=same, k1_TBps=r['k1_bytes_per_tick'] / sec / 1e12)
            r['k1_frac_of_hbm'] = r['k1_TBps'] * 1e12 / HBM_BPS
            print('round %d %-10s K1 %6.1f us  K2 %6.1f us  tick %6.1f us | K1 %.1f MB/tick  %.2f TB/s  %.0f %% of 3.35 TB/s | '
                  'outputs and state bit-identical to the first run: %s'
                  % (rnd, name, r['k1_us'], r['k2_us'], r['tick_us'], r['k1_bytes_per_tick'] / 1e6, r['k1_TBps'],
                     100 * r['k1_frac_of_hbm'], same), flush=True)
            results.append(r)
    for name, _, _ in arms:
        k1 = [r['k1_us'] for r in results if r['arm'] == name]
        tick = [r['tick_us'] for r in results if r['arm'] == name]
        print('%-10s K1 %.1f .. %.1f us   tick %.1f .. %.1f us' % (name, min(k1), max(k1), min(tick), max(tick)))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(dict(card=gpu, streams=S, prime=PRIME, timed=TIMED, results=results), f, indent=1)
    if not all(r['outputs_match_first'] for r in results):
        sys.exit('outputs differ between runs')


if __name__ == '__main__':
    main()
