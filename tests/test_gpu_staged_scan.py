"""-m gpu: the tick's window scan (gru_wg_kernel, rows staged from the MFCC ring through shared memory) against pb_predict on
the same windows (the same kernel, rows loaded directly from a [n][29][13] tensor).

Above 8 192 streams per tick both run the tensor-core scan with the same arithmetic (gru_wg_kernel<true, true> and
<false, true>), so a window scored by the tick and the same window read back (read_window) and scored by predict must
give bit-identical raw outputs.  This checks staging against direct loads, wgmma against itself; test_gpu_wg_scan.py
compares both with the mma.sync kernels.  A row staged from the wrong
ring slot, stream or step, or a zero row staged as data (or the reverse), shows up as a difference.  The ticks use permuted
subsets of the streams and clear some of them on the way, so windows start at every ring slot and young streams (fewer
than 29 frames, leading zero rows) are scored beside full ones."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')

from oracle import gru as og                      # noqa: E402


def test_staged_window_rows_match_direct_loads():
    import mycroft_precise_b200 as m
    # 2400-sample ticks release 3 frames each: 3 is prime to the 32-row ring, so window starts move through every slot
    S, K, chunk, ring_rows = 10000, 44, 2400, 32
    rs = np.random.RandomState(21)
    model = m.GruModel.random(13, 20, seed=3, scale=0.1)
    model.dense_b = 2.0
    w = og.GruWeights(model.kernel, model.recurrent, model.bias, model.dense_w, model.dense_b)
    sb = m.StreamBatch(model, S, chunk_samples=chunk)
    pr = sb.pr
    n_samples = np.zeros(S, np.int64)
    starts, young = set(), 0
    for k in range(K):
        if k in (12, 30):                                            # restart a quarter of the streams
            cl = np.sort(rs.choice(S, S // 4, replace=False)).astype(np.int32)
            sb.clear(torch.from_numpy(cl).cuda())
            n_samples[cl] = 0
        ids = rs.permutation(S)[:rs.randint(8500, S + 1)].astype(np.int32)
        pcm = np.clip(rs.randn(len(ids), chunk) * 3000, -32768, 32767).astype(np.int16)
        ids_t = torch.from_numpy(ids).cuda()
        raw = sb.update(torch.from_numpy(pcm).cuda(), ids_t)['raw'].clone()
        n_samples[ids] += chunk
        ns = n_samples[ids]
        released = np.where(ns >= pr.window_samples, (ns - pr.window_samples) // pr.hop_samples + 1, 0)
        full = released >= pr.n_features
        starts.update(((released[full] - pr.n_features) % ring_rows).tolist())
        young += int(np.count_nonzero(~full))

        wins = sb.core.read_window(ids=ids_t)
        direct = sb.core.predict(wins)
        assert torch.equal(direct, raw), 'tick %d: %d windows differ' % (k, int((direct != raw).sum()))
        p64 = og.gru_forward(w, wins.cpu().numpy(), np.float64)[0]
        assert np.max(np.abs(raw.cpu().numpy() - p64)) < 1e-5
    sb.core.close()
    assert starts == set(range(ring_rows)), sorted(starts)           # full windows start at every ring slot
    assert young > 0
