"""Stream audio history at the bench size (DESIGN.md §3 "Stream audio history", §6).

131 072 streams of the default geometry, a default-shaped network (H = 20 over 13 MFCCs) with seeded weights, seeded PCM.
  arm a: no history, update;
  arm b: buffer_samples (24 000) of history on every stream, update;
  arm c: the same history on 1 stream in 8 (a pool of S / 8 rows), update;
  arm d: arm b with ragged ticks, lengths 768..1280 at odd offsets, update_ragged.
The arms alternate in one process (REPS rounds); each round primes PRIME untimed ticks and times TIMED: K1 / K2 / the history
append from the library's CUDA-event profile (slots 0 / 1 / 3), the tick from CUDA events around the timed loop.  Byte model
of the append, per tick: for every item whose stream has history 2 len B of PCM read and 2 len B written into its row, plus
4 B of row map and 4 B of id read per item and 8 B of n_samples per history item.  a, b and c see the same ticks, so their
last tick's raw, conf, fired and counts must be bit-identical; b's last chunk must read back from its rows.

    python scripts/history_time.py [--out result.json]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np                      # noqa: E402
import torch                            # noqa: E402
import mycroft_precise_b200 as m        # noqa: E402
from bank_time import S, PRIME, TIMED, REPS, card   # noqa: E402


def timed(sb, tick, inputs):
    for i in range(PRIME):
        tick(inputs[i & 1])
    torch.cuda.synchronize()
    sb.core.profile(True)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for i in range(TIMED):
        out = tick(inputs[i & 1])
    t1.record()
    torch.cuda.synchronize()
    ms, launches = sb.core.profile_read()
    sb.core.profile(False)
    us = 1e3 / TIMED
    return dict(k1_us=ms[0] * us, k2_us=ms[1] * us, hist_us=ms[3] * us, hist_launches=int(launches[3]),
                tick_us=t0.elapsed_time(t1) * us), out


def same_bits(x, y):
    x, y = x.contiguous(), y.contiguous()
    return x.shape == y.shape and bool(torch.equal(x.view(torch.uint8), y.view(torch.uint8)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='also write the results as JSON to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('history_time.py needs a CUDA device')
    gpu = card()
    print('card:', gpu, flush=True)
    model = m.GruModel.random(13, 20, seed=0, scale=0.1)
    model.dense_b = 3.0                     # streams fire, so the counts compare something
    pcm_np = [np.clip(np.random.RandomState(i).randn(S, 1024) * 3000, -32768, 32767).astype(np.int16) for i in range(2)]
    pcm = [torch.from_numpy(x).cuda() for x in pcm_np]
    rs = np.random.RandomState(5)
    ragged = []
    for i in range(2):
        lens = rs.randint(768, 1281, S)
        off = np.concatenate([[1], 1 + np.cumsum(lens)]).astype(np.int64)          # odd offsets
        flat = np.clip(rs.randn(int(off[-1]) + 1) * 3000, -32768, 32767).astype(np.int16)
        ragged.append((torch.from_numpy(flat).cuda(), torch.from_numpy(off).cuda(), lens))
    a, b, c, d = (m.StreamBatch(model, S) for _ in range(4))
    B = a.pr.buffer_samples
    b.set_history(B)
    b.set_stream_history(True)
    c.set_history(B, max_rows=S // 8)
    c.set_stream_history(np.arange(S) % 8 == 0)
    d.set_history(B)
    d.set_stream_history(True)
    arms = [('a', a, a.update, pcm), ('b', b, b.update, pcm), ('c', c, c.update, pcm),
            ('d', d, lambda x: d.update_ragged(x[0], x[1], max_len=1280), ragged)]
    item = 4 + 4                            # row map + id per item
    model_bytes = dict(a=0, b=S * (4 * 1024 + item + 8), c=S * item + (S // 8) * (4 * 1024 + 8),
                       d=float(np.mean([4 * l.sum() for _, _, l in ragged])) + S * (item + 8))
    results = []
    for rep in range(REPS):
        row, outs = {}, {}
        for name, sb, tick, inputs in arms:
            sb.reset_count()
            row[name], o = timed(sb, tick, inputs)
            row[name]['append_tbs'] = model_bytes[name] / (row[name]['hist_us'] * 1e-6) / 1e12 if row[name]['hist_us'] else None
            outs[name] = {k: v.clone() for k, v in o.items()}
            print('round %d  %s  K1 %7.1f us  K2 %7.1f us  history %6.1f us (%d launches%s)  tick %7.1f us'
                  % (rep, name, row[name]['k1_us'], row[name]['k2_us'], row[name]['hist_us'], row[name]['hist_launches'],
                     ', %.2f TB/s' % row[name]['append_tbs'] if row[name]['append_tbs'] else '', row[name]['tick_us']),
                  flush=True)
        ok = all(same_bits(outs['a'][k], outs[x][k]) for x in 'bc' for k in ('raw', 'conf', 'fired'))
        ok = ok and same_bits(a.count, b.count) and same_bits(a.count, c.count)
        last = pcm_np[(TIMED - 1) & 1]
        back = b.read_history(torch.arange(64, dtype=torch.int32, device='cuda'), 1024).cpu().numpy()
        ok_read = bool(np.array_equal(back, last[:64]))
        print('round %d  a/b/c last tick and counts bit-identical: %s (count %d); b reads its last chunk back: %s'
              % (rep, ok, int(a.count.item()), ok_read), flush=True)
        assert ok and ok_read
        results.append(dict(round=rep, **row))
    print('byte model per tick: ' + ', '.join('%s %.1f MB' % (k, v / 1e6) for k, v in model_bytes.items()), flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(dict(card=gpu, streams=S, prime=PRIME, timed=TIMED, history_samples=B, byte_model=model_bytes,
                           results=results), f, indent=1)
    for x in (a, b, c, d):
        x.core.close()


if __name__ == '__main__':
    main()
