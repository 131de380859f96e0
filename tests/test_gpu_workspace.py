"""Every offline call on one handle, sharing its workspace: pb_score_corpus, pb_score_corpus_pool, pb_score_corpus_pairs,
pb_score_dataset, pb_vectorize_clips, pb_add_noise (with inputs), pb_generate (with windows), pb_train, pb_train_loss,
pb_train_wide and pb_score_rows.

The calls run twice in one sequence, small and large in turn, so the workspace grows in the middle of the sequence and later
calls reuse memory that another kind of call grew.  They alternate between the current stream and a side stream with no
synchronisation between them, so only the workspace's own ordering keeps one call from reusing memory another still reads.
Every output must equal the same call run alone on a fresh handle, bit for bit, and the handle's stream state must be
unchanged.  -m gpu."""
import numpy as np
import pytest

gpu = pytest.mark.gpu
TS, WS = 2980, 55812                          # PB_TRAIN_STRIDE, PB_TRAIN_WIDE_STRIDE
KINDS = ('corpus', 'corpus_pool', 'corpus_pairs', 'dataset', 'vectorize', 'noise', 'generate', 'train', 'train_loss',
         'train_wide', 'rows')


def _sig(n, seed, sigma=3000):
    rs = np.random.RandomState(seed)
    return np.clip(np.round(rs.randn(n) * sigma), -32768, 32767).astype(np.int16)


def _pack(torch, recs, lead=3):
    """Recordings back to back after `lead` samples (odd offsets, so both K1 paths run): (tensor, offsets)."""
    pcm = np.concatenate([_sig(lead, 999)] + list(recs))
    offsets = lead + np.concatenate([[0], np.cumsum([len(r) for r in recs])]).astype(np.int64)
    return torch.from_numpy(pcm).cuda(), offsets


def _rows(m, core, hidden, stride, seed):
    """Training rows of random networks (from_models' layout at `stride`): (train_rows' array, weights, rms)."""
    import torch
    acts = [('linear', 'hard_sigmoid'), ('tanh', 'sigmoid')]
    w = np.zeros((len(hidden), stride), np.float32)
    for i, H in enumerate(hidden):
        g = m.GruModel.random(core.feature_size, H, seed=seed + i, scale=0.1)
        flat = np.concatenate([g.kernel.ravel(), g.recurrent.ravel(), g.bias, g.dense_w, [np.float32(g.dense_b)]])
        w[i, :flat.size] = flat
    rows = core.train_rows(hidden, [acts[i % 2][0] for i in range(len(hidden))], [acts[i % 2][1] for i in range(len(hidden))],
                           [seed + i for i in range(len(hidden))])
    return rows, torch.from_numpy(w).cuda(), torch.zeros((len(hidden), stride), device='cuda')


class Case:
    """Every call's arguments at one size (0 small, 1 large)."""

    def __init__(self, m, core, size):
        import torch
        from mycroft_precise_b200.core import GEN_ITEM, GEN_SEGMENT
        rs = np.random.RandomState(10 + size)
        n = (12, 120)[size]
        self.n = n
        self.clips = [_sig(int(L), 100 * size + i) for i, L in enumerate(rs.randint(800, 40000, n))]
        self.pcm, self.offsets = _pack(torch, self.clips)
        self.targets = (rs.rand(n) < 0.4).astype(np.uint8)
        k = (3, 12)[size]
        self.ids = (np.arange(k) % 6).astype(np.int32)
        n_pairs = (20, 400)[size]
        self.pair_models = rs.randint(0, 6, n_pairs).astype(np.int32)
        self.pair_recs = rs.randint(0, n, n_pairs).astype(np.int32)
        self.noise = torch.from_numpy(_sig(50000 + 17 * size, 7)).cuda()
        n_items = (10, 150)[size]
        self.noise_items = rs.randint(0, n, n_items).astype(np.int32)
        self.ratios = rs.rand(n_items)
        # generated streams: clip stretches and silence over backgrounds, windows on every third chunk
        bgs = [_sig(60000 + 1000 * b, 200 + b, 2000) for b in range(3)]
        self.bg, self.bg_offsets = _pack(torch, bgs)
        self.gen_clips, self.gen_clip_offsets = self.pcm, self.offsets
        items, segs, wins = [], [], []
        for i in range((8, 60)[size]):
            b, L = i % 3, int(rs.randint(3000, 60000))
            s0 = len(segs)
            c = int(rs.randint(0, n))
            segs += [(-1, 0, 0, int(rs.randint(0, 5000))), (c, 0, 0, len(self.clips[c])), (-1, 0, 0, L)]
            items.append((b, 0, 0.4 + 0.5 * rs.rand(), L, s0, len(segs)))
            wins += [(i, ch) for ch in range(0, L // 2048, 3)]
        self.gen_items = np.array(items, GEN_ITEM)
        self.gen_segs = np.array(segs, GEN_SEGMENT)
        self.gen_windows = np.array(wins, np.int64)
        # training: vectorized clips (on a handle of their own), fused and wide rows
        v = m.PreciseB200()
        self.inputs = v.vectorize_clips(self.pcm, self.offsets)
        torch.cuda.synchronize()
        v.close()
        kt = (3, 16)[size]
        self.fused = _rows(m, core, [int(h) for h in rs.randint(1, 25, kt)], TS, 500 + size)
        self.wide = _rows(m, core, [int(h) for h in rs.randint(1, 129, kt)], WS, 700 + size)
        self.rows_pairs = (rs.randint(0, kt, 3 * n).astype(np.int32), rs.randint(0, n, 3 * n).astype(np.int32))


def _run(kind, core, c):
    """One call of `kind` on `core` with case `c`, on the current stream: its outputs (device tensors, none waited for)."""
    if kind == 'corpus':
        o = core.score_corpus(c.pcm, c.offsets)
        return [o['raw'], o['conf'], o['fired'], o['activations']]
    if kind == 'corpus_pool':
        o = core.score_corpus_pool(c.pcm, c.offsets, c.ids, schedule='simulate', chunk=2048)
        return [o['raw'], o['conf'], o['fired'], o['activations'], o['above'], o['sum']]
    if kind == 'corpus_pairs':
        o = core.score_corpus_pairs(c.pcm, c.offsets, c.pair_models, c.pair_recs)
        return [o['raw'], o['conf'], o['fired'], o['activations']]
    if kind == 'dataset':
        a = core.score_dataset(c.pcm, c.offsets, c.targets, c.ids)
        rows = (c.pair_models % len(c.ids)).astype(np.int32)
        b = core.score_dataset(c.pcm, c.offsets, c.targets, c.ids, rows=rows, recs=c.pair_recs, per_entry=False)
        return [a['raw'], a['count'], a['hist'], a['fit'], b['count'], b['hist'], b['fit']]
    if kind == 'vectorize':
        return [core.vectorize_clips(c.pcm, c.offsets)]
    if kind == 'noise':
        return list(core.add_noise(c.pcm, c.offsets, c.noise, c.noise_items, c.ratios, noise_pos=11, inputs=True))
    if kind == 'generate':
        return list(core.generate(c.bg, c.bg_offsets, c.gen_clips, c.gen_clip_offsets, c.gen_items, c.gen_segs,
                                  windows=c.gen_windows))
    if kind in ('train', 'train_wide'):
        rows, w, rms = c.fused if kind == 'train' else c.wide
        w, rms = w.clone(), rms.clone()
        loss = core.train(c.inputs, c.targets, rows, w, rms, epochs=2, batch_size=64)
        return [loss, w, rms]
    if kind == 'train_loss':
        rows, w, _ = c.fused
        return list(core.train_loss(c.inputs, c.targets, rows, w, dropout=0.2, epoch=3, grad=True))
    rows, w, _ = c.wide
    a = core.score_rows(c.inputs, c.targets, rows, w)
    b = core.score_rows(c.inputs, c.targets, rows, w, pair_rows=c.rows_pairs[0], pair_recs=c.rows_pairs[1])
    return [a['raw'], a['count'], a['hist'], a['fit'], b['raw'], b['count'], b['hist'], b['fit']]


def _handle(m, models):
    core = m.PreciseB200()
    core.load_weights(models[0].kernel, models[0].recurrent, models[0].bias, models[0].dense_w, models[0].dense_b)
    core.set_pool(len(models))
    for i, g in enumerate(models):
        core.pool_load(i, g)
    return core


@gpu
def test_every_offline_call_shares_one_workspace_across_streams():
    torch = pytest.importorskip('torch')
    import mycroft_precise_b200 as m
    models = []
    for i in range(6):
        g = m.GruModel.random(13, [20, 12, 24, 16, 8, 20][i], seed=40 + i, scale=0.1)
        if i % 3 == 2:
            g.activation, g.recurrent_activation = 'tanh', 'sigmoid'
        g.dense_b = 1.5 - 0.5 * i
        models.append(g)
    core = _handle(m, models)
    cases = [Case(m, core, 0), Case(m, core, 1)]
    # kind i runs at size (i // 2 + r) % 2 in round r: both sizes and both streams for every kind, growth mid-sequence
    seq = [(kind, (i // 2 + r) % 2) for r in range(2) for i, kind in enumerate(KINDS)]

    alone = {}
    for kind, size in set(seq):
        fresh = _handle(m, models)
        alone[kind, size] = [t.cpu().numpy() for t in _run(kind, fresh, cases[size])]
        torch.cuda.synchronize()
        fresh.close()

    state = core.export_streams().cpu().numpy()
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    got = []
    for j, (kind, size) in enumerate(seq):
        with torch.cuda.stream(side if j % 2 else torch.cuda.current_stream()):
            got.append(_run(kind, core, cases[size]))
    torch.cuda.synchronize()
    for (kind, size), outs in zip(seq, got):
        ref = alone[kind, size]
        assert len(outs) == len(ref)
        for q, (a, b) in enumerate(zip(outs, ref)):
            a = a.cpu().numpy()
            assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), (kind, size, q)
    assert np.array_equal(core.export_streams().cpu().numpy(), state)
    core.close()
