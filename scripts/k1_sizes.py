"""K1 time of the FFT kernel with its 32-bit (mode 0) and 64-bit (mode 3) set-up over batch sizes."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch, mycroft_precise_b200 as m
model = m.GruModel.random(13, 20, seed=0, scale=0.1)
for S in [int(a) for a in sys.argv[1:]] or [4096, 16384, 32768, 65536, 131072, 262144]:
    pcm = torch.from_numpy((np.random.RandomState(0).randn(S, 1024) * 3000).astype(np.int16)).cuda()
    res = []
    for mode in (0, 3):
        sb = m.StreamBatch(model, S, chunk_samples=1024)
        sb.core.k1_mode(mode)
        for _ in range(30):
            sb.update(pcm)
        torch.cuda.synchronize()
        sb.core.profile(True)
        for _ in range(20):
            sb.update(pcm)
        ms, n = sb.core.profile_read()
        res.append(1e3 * ms[0] / n[0])
        sb.core.close()
    print('S %7d  FFT %.1f us  tc3 %.1f us  ratio %.2f' % (S, res[0], res[1], res[0] / res[1]), flush=True)
