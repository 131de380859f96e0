"""The pipelined stateful MFCC kernel (k1 mode 0, mfcc_pipe_stream_kernel) against the kernel it replaced (k1 mode 2,
mfcc_fast_stream_kernel<true>): two handles take the same ticks, and after every tick raw, conf, fired and every stream's
exported state (MFCC ring, tail, n_samples, network and trigger state) must be equal bit for bit.

Covers batch sizes around the tile and warp boundaries (one stream per warp up to 2 112 streams on 132 SMs, 16-stream tiles
at 131 072), id subsets and permutations, streams of mixed ages (cleared mid-run, imported), a handle with a history pool, and
chunks of 512 (the short-chunk tail shift), 800, 1 024 and 4 096 samples.  6 400-sample chunks complete more than 8 frames per
stream, so both modes run them through the generic kernel: that case checks that mode 0 leaves it alone.
"""
import numpy as np
import pytest

from test_gpu_stream_models import cuda, host, noise
from test_gpu_stream_trigger import hot_model

gpu = pytest.mark.gpu


def _mod():
    import mycroft_precise_b200 as m
    return m


def same(x, y):
    x, y = np.ascontiguousarray(x), np.ascontiguousarray(y)
    return x.shape == y.shape and np.array_equal(x.view(np.uint8), y.view(np.uint8))


def handles(m, S, chunk, history=False):
    model = hot_model(m, seed=5)
    new, old = m.StreamBatch(model, S, chunk_samples=chunk), m.StreamBatch(model, S, chunk_samples=chunk)
    old.core.k1_mode(2)
    if history:
        for sb in (new, old):
            sb.set_history(max_rows=S)
            sb.set_stream_history(np.arange(S) % 3 == 0)
    return new, old


def tick_both(new, old, pcm, ids):
    g = None if ids is None else cuda(ids)
    on, oo = host(new.update(cuda(pcm), g)), host(old.update(cuda(pcm), g))
    for x, y in zip(on, oo):
        assert same(x, y)
    assert same(new.core.export_streams().cpu().numpy(), old.core.export_streams().cpu().numpy())


def run(new, old, S, n, chunk, K, rs, clear_at=None):
    """K ticks of n items: the first tick in id order (ids None when n == S), then random subsets in random order."""
    for k in range(K):
        if k == 0:
            ids = None if n == S else np.arange(n, dtype=np.int32)
        else:
            ids = rs.permutation(S)[:n].astype(np.int32)
        tick_both(new, old, noise((n, chunk), rs), ids)
        if clear_at is not None and k == clear_at:
            c = cuda(rs.permutation(S)[:max(1, S // 4)].astype(np.int32))
            new.core.clear(ids=c)
            old.core.clear(ids=c)


@gpu
@pytest.mark.parametrize('n', [1, 15, 17, 1000, 33791, 33797])
def test_batch_sizes_subsets_and_clears(n):
    m = _mod()
    S = n + n // 3 + 1
    new, old = handles(m, S, 1024)
    run(new, old, S, n, 1024, 6, np.random.RandomState(n), clear_at=2)
    for sb in (new, old):
        sb.core.close()


@gpu
@pytest.mark.parametrize('chunk', [512, 800, 1024, 4096, 6400])
@pytest.mark.parametrize('n', [17, 1000])
def test_chunks(chunk, n):
    m = _mod()
    S = n + 5
    new, old = handles(m, S, chunk)
    run(new, old, S, n, chunk, 8 if chunk < 1024 else 5, np.random.RandomState(chunk + n), clear_at=3)
    for sb in (new, old):
        sb.core.close()


@gpu
def test_every_warp_walks_several_tiles():
    m = _mod()
    S = 131072
    new, old = handles(m, S, 1024)
    run(new, old, S, S, 1024, 4, np.random.RandomState(3))
    for sb in (new, old):
        sb.core.close()


@gpu
def test_imported_streams_and_history():
    """Streams of mixed ages imported from a third handle into both, on handles with a history pool."""
    m = _mod()
    S, n = 3000, 2500
    rs = np.random.RandomState(11)
    src = m.StreamBatch(hot_model(m, seed=5), S)
    for k in range(7):
        sids = rs.permutation(S)[:rs.randint(S // 3, S)].astype(np.int32)
        src.update(cuda(noise((len(sids), 1024), rs)), cuda(sids))
    snap = src.export_streams()
    new, old = handles(m, S, 1024, history=True)
    run(new, old, S, n, 1024, 2, rs)
    dst = rs.permutation(S)[:S // 2].astype(np.int32)
    part = dict(snap, state=snap['state'][:S // 2], stream_models=snap['stream_models'][:S // 2],
                stream_trigger=[tuple(a[:S // 2] for a in t) for t in snap['stream_trigger']])
    for sb in (new, old):
        sb.import_streams(part, dst)
    run(new, old, S, n, 1024, 5, rs)
    for sb in (new, old, src):
        sb.core.close()
