"""K2 A/B at the bench size (pb_debug_gru_mode): 0 = default (fp16x3 scan, staged projection blocks, projects its own new frames, 4 CTAs/SM),
11 = the same at 5 CTAs/SM, 10 = 3xTF32 staged, 9 = 3xTF32 with LDG loads, 7 = 3xTF32 32-stream tiles."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch, mycroft_precise_b200 as m
S = 131072
modes = [int(a) for a in sys.argv[1:]] or [0, 10, 9]
model = m.GruModel.random(13, 20, seed=0, scale=0.1)
pcm = [torch.from_numpy((np.random.RandomState(i).randn(S, 1024) * 3000).astype(np.int16)).cuda() for i in range(2)]
for mode in modes:
    sb = m.StreamBatch(model, S, chunk_samples=1024)
    sb.core.gru_mode(mode)
    for i in range(30):
        sb.update(pcm[i & 1])
    torch.cuda.synchronize()
    sb.core.profile(True)
    for i in range(20):
        sb.update(pcm[i & 1])
    ms, n = sb.core.profile_read()
    print('gru_mode', mode, 'K1 %.1f us' % (1e3 * ms[0] / n[0]), 'K2 %.1f us' % (1e3 * ms[1] / n[1]), 'proj %.1f us' % (1e3 * ms[3] / max(1, n[3])), flush=True)
    sb.core.close()
