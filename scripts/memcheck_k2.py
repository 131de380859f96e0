"""Small run of the default large-batch tick (MFCC kernels + gru_bank_kernel, a partial last tile, shuffled ids) for compute-sanitizer."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch, mycroft_precise_b200 as m
S = 9000 + 7
model = m.GruModel.random(13, 20, seed=0, scale=0.1)
sb = m.StreamBatch(model, S, chunk_samples=1024)
rs = np.random.RandomState(0)
ids = torch.from_numpy(rs.permutation(S)[:8500].astype(np.int32)).cuda()
for k in range(5):
    pcm = torch.from_numpy((rs.randn(S, 1024) * 3000).astype(np.int16)).cuda()
    if k == 3:
        sb.update(pcm[:8500], ids)          # shuffled ids: a tile's 16 streams are scattered over the ring
    else:
        sb.update(pcm)
torch.cuda.synchronize()
print('ok', int(sb.count.item()))
