"""The pipelined stateful MFCC kernel (k1 mode 0) compiles the default front end's mel shape in (mel16_fixed: 3 piece blocks, at
most 9 slots per filter, 20 filters, 13 MFCCs) and runs every other shape through its table-driven instantiation (mel16).
Both must stay bit-identical to mode 2 (mfcc_fast_stream_kernel<true>) in raw, conf, fired and every stream's exported state,
at batch sizes around the warp count of the grid (fewer 16-stream tiles than warps, as many, one more, and 3 x warps + 272:
131 072 streams on 132 SMs) and on id subsets in random order.
"""
import numpy as np
import pytest

from test_gpu_k1_pipeline import handles, tick_both
from test_gpu_stream_models import noise

gpu = pytest.mark.gpu

K1P_CTAS_PER_SM, K1F_WARPS, SPW = 5, 4, 16


def _mod():
    import mycroft_precise_b200 as m
    return m


def pipe_warps():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * K1P_CTAS_PER_SM * K1F_WARPS


def ticks(new, old, S, n, K, rs):
    for k in range(K):
        ids = None if (k == 0 and n == S) else rs.permutation(S)[:n].astype(np.int32)
        tick_both(new, old, noise((n, 1024), rs), ids)


@gpu
@pytest.mark.parametrize('case', ['fewer_tiles', 'tiles_eq_warps', 'warps_plus_1', '3warps_plus_272'])
def test_default_shape_tile_counts(case):
    m = _mod()
    w = pipe_warps()
    tiles = {'fewer_tiles': w // 2 + 1, 'tiles_eq_warps': w, 'warps_plus_1': w + 1, '3warps_plus_272': 3 * w + 272}[case]
    n = tiles * SPW                          # below 16 x 4 warps per SM the tiles shrink: 'fewer_tiles' stays below w tiles
    S = n + n // 7 + 3
    new, old = handles(m, S, 1024)
    ticks(new, old, S, n, 3, np.random.RandomState(tiles))
    for sb in (new, old):
        sb.core.close()


@gpu
@pytest.mark.parametrize('shape', ['mfcc40', 'mfcc12'])
def test_other_mel_shapes(shape):
    m = _mod()
    kw = {'mfcc40': dict(n_filt=40, n_mfcc=40), 'mfcc12': dict(n_mfcc=12)}[shape]
    model = m.GruModel.random(kw['n_mfcc'], 20, seed=9, scale=0.1)
    model.dense_b = 3.0
    w = pipe_warps()
    n = (w + 301) * SPW
    S = n + n // 5
    new, old = (m.StreamBatch(model, S, params=m.ListenerParams(**kw), chunk_samples=1024) for _ in range(2))
    old.core.k1_mode(2)
    ticks(new, old, S, n, 4, np.random.RandomState(len(shape)))
    for sb in (new, old):
        sb.core.close()
