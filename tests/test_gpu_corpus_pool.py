"""Pool models over recorded corpora (pb_score_corpus_pool, offline.score_corpus_pool / simulate_pool, precise-simulate with
several models).  The reference for every pool row is the same network in a bank of two fused models scored by
pb_score_corpus on the same recordings: every output must be equal bit for bit.  -m gpu except the command-line checks that
need no device."""
import ctypes as C
import os
import re
import subprocess
import sys
import wave

import numpy as np
import pytest

from oracle import gru as og
from oracle.listener import OracleListener
from oracle.params import OracleParams
from oracle.trigger import OracleTrigger

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ('raw', 'conf', 'fired', 'activations', 'above', 'sum')
CONFIGS = [('listener', 1024), ('listener', 2048), ('simulate', 4096), ('simulate', 1600)]


def _mod():
    import mycroft_precise_b200 as m
    return m


def _noise(n, seed, sigma=3000):
    rs = np.random.RandomState(seed)
    return np.clip(rs.randn(n) * sigma * (1 + np.sin(np.arange(n) / 4000.0)), -32768, 32767).astype(np.int16)


def pool_models(m):
    """(model, params, sensitivity, trigger_level) of twelve fused networks: H = 8 .. 24, Keras's and tanh / sigmoid
    activations, one with its own threshold_config and center, varied triggers; dense biases make them fire."""
    m0 = m.GruModel.random(13, 20, seed=0, scale=0.1)
    m1 = m.GruModel.random(13, 12, seed=1, scale=0.1)
    m2 = m.GruModel.random(13, 20, seed=2, scale=0.1)
    m2.activation, m2.recurrent_activation = 'tanh', 'sigmoid'
    p1 = m.ListenerParams(threshold_config=((8, 3),), threshold_center=0.3)
    spec = [(m0, None, 0.8, 1), (m1, p1, 0.8, 1), (m2, None, 0.5, 3)]
    for i in range(9):
        g = m.GruModel.random(13, [20, 12, 24, 16, 8][i % 5], seed=100 + i, scale=0.1)
        if i % 3 == 2:
            g.activation, g.recurrent_activation = 'tanh', 'sigmoid'
        spec.append((g, None, 0.5 + 0.1 * (i % 4), 1 + i % 3))
    for i, (g, pr, _, _) in enumerate(spec):
        g.dense_b = (pr.threshold_config[0][0] if pr is not None else 3.0) - 0.5 * (i % 3)
    return spec


def corpus():
    """Recordings packed back to back from offset 0, so some start off a multiple of 8 samples (the generic K1): empty,
    shorter than a window, exactly one chunk of 1024 and of 4096, lengths that are not multiples of 8, silence, full-scale
    DC, about 60 s of noise."""
    recs = [np.zeros(0, np.int16), _noise(100, 1), _noise(1024, 2), _noise(4096, 3), _noise(24801, 4), _noise(3333, 5),
            np.zeros(20000, np.int16), np.full(20000, 32767, np.int16), _noise(16000 * 60 + 3, 6)]
    offsets = np.concatenate([[0], np.cumsum([len(r) for r in recs])]).astype(np.int64)
    return recs, np.concatenate(recs), offsets


class Fixture:
    def __init__(self):
        import torch
        m = _mod()
        self.m = m
        self.spec = pool_models(m)
        self.recs, pcm, self.offsets = corpus()
        self.pcm = torch.from_numpy(pcm).cuda()
        self.pool = m.PreciseB200()
        self.pool.set_pool(len(self.spec))
        for i, (model, pr, sens, lvl) in enumerate(self.spec):
            self.pool.pool_load(i, model, pr, sensitivity=sens, trigger_level=lvl)
        # model i is slot 1 of a bank of two (slot 0: the default-shaped network of spec[0])
        m0 = self.spec[0][0]
        self.banks = []
        for model, pr, sens, lvl in self.spec:
            b = m.PreciseB200()
            b.load_weights(m0.kernel, m0.recurrent, m0.bias, m0.dense_w, m0.dense_b)
            b.add_model(model, pr, sensitivity=sens, trigger_level=lvl)
            self.banks.append(b)
        self._ref = {}

    def ref(self, schedule, chunk, divisor=32768, threshold=0.5):
        """{key: [12][...] host arrays} of the bank rows."""
        key = (schedule, chunk, divisor, threshold)
        if key not in self._ref:
            rows = {k: [] for k in KEYS}
            for b in self.banks:
                r = b.score_corpus(self.pcm, self.offsets, schedule, chunk, threshold, divisor)
                for k in KEYS:
                    rows[k].append(None if r[k] is None else r[k][1].cpu().numpy())
            self._ref[key] = rows
        return self._ref[key]

    def close(self):
        self.pool.close()
        for b in self.banks:
            b.close()


@pytest.fixture(scope='module')
def fx():
    pytest.importorskip('torch')
    f = Fixture()
    yield f
    f.close()


def _host(res):
    return {k: None if res[k] is None else res[k].cpu().numpy() for k in KEYS}


def _same(a, b):
    """Bit-identical (NaN included)."""
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def _check_rows(got, ref, ids, keys=KEYS):
    for k in keys:
        if ref[k][0] is None:
            assert got[k] is None, k
            continue
        assert got[k].shape[0] == len(ids), k
        for i, mid in enumerate(ids):
            assert _same(got[k][i], ref[k][mid]), (k, i, mid)


@gpu
@pytest.mark.parametrize('schedule,chunk', CONFIGS)
@pytest.mark.parametrize('divisor', [32768, 32767])
def test_bit_identity(fx, schedule, chunk, divisor):
    ids = np.arange(len(fx.spec), dtype=np.int32)
    got = _host(fx.pool.score_corpus_pool(fx.pcm, fx.offsets, ids, schedule, chunk, 0.5, divisor))
    ref = fx.ref(schedule, chunk, divisor)
    _check_rows(got, ref, ids)
    assert got['raw'].shape[1] >= fx.pool.corpus_windows(len(fx.recs[-1]), schedule, chunk)   # the 60 s recording is there
    assert got['activations'].sum() > 0                         # the models fire


@gpu
@pytest.mark.parametrize('nm,groups_fast', [(0, -1), (1, 1), (2, 0), (4, 1), (8, 1), (8, 0)])
def test_model_lists(fx, nm, groups_fast):
    """k = 1, 7, 9, 12 (partial groups for every NM), a permutation interleaving the activation classes, repeated ids, with
    every scan shape and grid order."""
    fx.pool.corpus_pool_scan(nm, groups_fast)
    try:
        lists = [[5], list(range(7)), list(range(3, 12)), list(range(12)),
                 [2, 0, 5, 11, 8, 1, 4, 3, 10, 7, 6, 9], [4, 4, 2, 4, 0, 2, 2, 11, 11]]
        for schedule, chunk in (CONFIGS[0], CONFIGS[2]):
            ref = fx.ref(schedule, chunk)
            for ids in lists:
                ids = np.asarray(ids, np.int32)
                got = _host(fx.pool.score_corpus_pool(fx.pcm, fx.offsets, ids, schedule, chunk))
                _check_rows(got, ref, ids)
    finally:
        fx.pool.corpus_pool_scan(0, -1)


@gpu
def test_subset_of_larger_pool(fx):
    """A pool of 40 slots with the twelve models spread out between empty slots; a request of a subset of them."""
    m = fx.m
    core = m.PreciseB200()
    core.set_pool(40)
    slot = [3 * i + 1 for i in range(len(fx.spec))]
    for i, (model, pr, sens, lvl) in enumerate(fx.spec):
        core.pool_load(slot[i], model, pr, sensitivity=sens, trigger_level=lvl)
    want = [9, 2, 7, 0, 11]
    ids = np.asarray([slot[i] for i in want], np.int32)
    for schedule, chunk in (CONFIGS[1], CONFIGS[3]):
        got = _host(core.score_corpus_pool(fx.pcm, fx.offsets, ids, schedule, chunk))
        _check_rows(got, fx.ref(schedule, chunk), want)
    core.close()


@gpu
@pytest.mark.parametrize('schedule,chunk', [CONFIGS[0], CONFIGS[2]])
def test_reductions_only_and_batches(fx, schedule, chunk):
    """per_window=False gives the reductions of a per_window=True call; at most 1 or 3 rows per batch (several batches and a
    short last one) give them again."""
    ids = np.asarray([2, 0, 5, 11, 8, 1, 4, 3, 10, 7, 6, 9, 0], np.int32)
    full = _host(fx.pool.score_corpus_pool(fx.pcm, fx.offsets, ids, schedule, chunk))
    red = ('activations', 'above', 'sum')
    try:
        for rows in (0, 1, 3):
            fx.pool.corpus_pool_rows(rows)
            got = _host(fx.pool.score_corpus_pool(fx.pcm, fx.offsets, ids, schedule, chunk, per_window=False))
            assert got['raw'] is None and got['conf'] is None and got['fired'] is None
            for k in red:
                if full[k] is None:
                    assert got[k] is None
                else:
                    assert _same(got[k], full[k]), (rows, k)
    finally:
        fx.pool.corpus_pool_rows(0)
    # each output alone
    lib, h = fx.pool.lib, fx.pool._h
    import torch
    W, n = full['raw'].shape[1], len(fx.offsets) - 1
    k = len(ids)
    sched = 0 if schedule == 'listener' else 1
    for name, shape, dt in (('raw', (k, W), torch.float32), ('conf', (k, W), torch.float64), ('fired', (k, W), torch.uint8),
                            ('activations', (k, n), torch.int64)):
        t = torch.empty(shape, dtype=dt, device='cuda')
        args = {x: None for x in KEYS}
        args[name] = C.c_void_p(t.data_ptr())
        rc = lib.pb_score_corpus_pool(h, C.c_void_p(fx.pcm.data_ptr()), fx.offsets.ctypes.data_as(C.c_void_p), n,
                                      ids.ctypes.data_as(C.c_void_p), k, 32768, sched, chunk, 0.5,
                                      *[args[x] for x in KEYS], None)
        assert rc == 0
        assert _same(t.cpu().numpy(), full[name]), name


def _oracle_listener(model, pr, a, c, sensitivity, trigger_level):
    opr = OracleParams(**(pr.to_dict() if pr is not None else {}))
    w = og.GruWeights(model.kernel, model.recurrent, model.bias, model.dense_w, model.dense_b,
                      activation=model.activation, recurrent_activation=model.recurrent_activation)
    lis = OracleListener(w, opr)
    K = len(a) // c
    raw = np.zeros(K, np.float32)
    for k in range(K):
        raw[k] = lis.update_raw(a[k * c:(k + 1) * c].astype(np.float32) / np.float32(32768))
    return raw


@gpu
def test_oracle_anchor(fx):
    """Two models (the default network and the tanh / sigmoid one): raw against the oracle listener on its own windows;
    fired equals OracleTrigger replayed on the library's conf."""
    c = 1024
    ids = np.asarray([0, 2], np.int32)
    got = fx.pool.score_corpus_pool(fx.pcm, fx.offsets, ids, 'listener', c)
    wo = np.concatenate([[0], np.cumsum([len(a) // c for a in fx.recs])])
    raw, conf, fired = (got[k].cpu().numpy() for k in ('raw', 'conf', 'fired'))
    worst = 0.0
    for row, mid in enumerate(ids):
        model, pr, sens, lvl = fx.spec[mid]
        for i, a in enumerate(fx.recs):
            sl = slice(wo[i], wo[i + 1])
            want = _oracle_listener(model, pr, a, c, sens, lvl)
            if want.size:
                worst = max(worst, float(np.max(np.abs(raw[row, sl] - want))))
            det = OracleTrigger(2 * c, sens, lvl)
            assert [bool(det.update(float(x))) for x in conf[row, sl]] == list(fired[row, sl].astype(bool)), (mid, i)
    print('max |raw - oracle| = %.3g' % worst)
    assert worst < 1e-5, worst
    assert fired.sum() > 0


@gpu
def test_no_side_effects(fx):
    """Corpus calls interleaved with combined and pool ticks leave the ticks and the stream assignments as a twin handle
    without them has them; a pool_load right after a queued call leaves that call's rows the old model's."""
    import torch
    m = fx.m
    S, K, chunk = 6, 8, 1024
    twins = []
    for _ in range(2):
        sb = m.StreamBatch(fx.spec[0][0], S, chunk_samples=chunk)
        sb.set_pool(len(fx.spec))
        for i, (model, pr, sens, lvl) in enumerate(fx.spec):
            sb.pool_load(i, model, pr, sensitivity=sens, trigger_level=lvl)
        sb.set_stream_pool(np.asarray([0, 2, 5, -1, 7, 2], np.int32))
        sb.set_stream_pool_trigger(0.7, 1, 4096, ids=np.asarray([1, 4], np.int32))
        twins.append(sb)
    rs = np.random.RandomState(3)
    pcm = [torch.from_numpy(np.clip(rs.randn(S, chunk) * 3000, -32768, 32767).astype(np.int16)).cuda() for _ in range(K)]
    outs = [[], []]
    ids = np.arange(len(fx.spec), dtype=np.int32)
    ref = fx.ref('listener', 1024)
    for k in range(K):
        for t, sb in enumerate(twins):
            o = sb.update_all(pcm[k]) if k % 2 else sb.update_pool(pcm[k])
            outs[t].append({x: o[x].cpu().numpy() for x in ('raw', 'conf', 'fired')})
            if t == 0:
                got = _host(sb.core.score_corpus_pool(fx.pcm, fx.offsets, ids, 'listener', 1024))
                _check_rows(got, ref, ids)
    for a, b in zip(*outs):
        for x in a:
            assert _same(a[x], b[x]), x
    assert np.array_equal(twins[0].core.stream_pool(), twins[1].core.stream_pool())
    assert int(twins[0].pool_count.item()) == int(twins[1].pool_count.item())
    # a load issued right after a queued call
    core = twins[0].core
    res = core.score_corpus_pool(fx.pcm, fx.offsets, np.asarray([3, 3], np.int32), 'listener', 1024)
    core.pool_load(3, fx.spec[4][0], fx.spec[4][1], sensitivity=fx.spec[4][2], trigger_level=fx.spec[4][3])
    _check_rows(_host(res), ref, [3, 3])
    got = _host(core.score_corpus_pool(fx.pcm, fx.offsets, np.asarray([3], np.int32), 'listener', 1024))
    _check_rows(got, ref, [4])
    for sb in twins:
        sb.core.close()


@gpu
def test_refusals(fx):
    import torch
    from mycroft_precise_b200.core import PBError
    m = fx.m
    core = fx.pool
    lib, h = core.lib, core._h
    ids = np.arange(4, dtype=np.int32)
    before = _host(core.score_corpus_pool(fx.pcm, fx.offsets, ids, 'simulate', 4096))
    n = len(fx.offsets) - 1
    act = torch.zeros((4, n), dtype=torch.int64, device='cuda')

    def call(model_ids, k, outs=True, divisor=32768, schedule=1, chunk=4096, offsets=fx.offsets):
        p_ids = None if model_ids is None else model_ids.ctypes.data_as(C.c_void_p)
        return lib.pb_score_corpus_pool(h, C.c_void_p(fx.pcm.data_ptr()), offsets.ctypes.data_as(C.c_void_p), n, p_ids, k,
                                        divisor, schedule, chunk, 0.5, None, None, None,
                                        C.c_void_p(act.data_ptr()) if outs else None, None, None, None)

    assert call(ids, -1) == -1                                                 # k < 0
    assert call(None, 4) == -1                                                 # null ids
    assert call(np.asarray([0, 12], np.int32), 2) == -1                        # outside [0, max_models)
    assert call(np.asarray([-1], np.int32), 1) == -1
    assert call(ids, 4, outs=False) == -1                                      # every output null
    assert call(ids, 4, divisor=1000) == -1
    assert call(ids, 4, schedule=7) == -1
    assert call(ids, 4, chunk=10) == -1                                        # simulate chunk below one hop
    assert call(ids, 4, offsets=fx.offsets[::-1].copy()) == -1                 # decreasing offsets
    assert call(ids, 0) == 0                                                   # nothing to score
    with pytest.raises(ValueError, match='holds no model'):
        empty = m.PreciseB200()
        empty.set_pool(4)
        empty.pool_load(0, fx.spec[0][0])
        empty.score_corpus_pool(fx.pcm, fx.offsets, np.asarray([0, 1], np.int32), 'simulate', 4096)
    empty.close()
    nopool = m.PreciseB200()
    with pytest.raises(PBError, match='no model pool'):
        nopool.score_corpus_pool(fx.pcm, fx.offsets, ids, 'simulate', 4096)
    nopool.close()
    with pytest.raises(ValueError):
        core.score_corpus_pool(fx.pcm, fx.offsets, ids, 'listener', 1024, per_window=True, divisor=12)
    assert not act.any()                                                       # refused calls wrote nothing
    after = _host(core.score_corpus_pool(fx.pcm, fx.offsets, ids, 'simulate', 4096))
    for k in KEYS:
        assert (before[k] is None and after[k] is None) or _same(before[k], after[k]), k


@gpu
def test_simulate_pool_matches_simulate(fx):
    """Totals bit-identical to offline.score_corpus's bank row of the same network, and equal to offline.simulate on a
    one-model handle (whose scan may be another kernel: counts equal, sums to 1e-6)."""
    from mycroft_precise_b200 import offline
    m = fx.m
    recs = fx.recs + [_noise(40000, 9)]
    ids = np.asarray([1, 0, 2, 6, 10], np.int32)
    metrics, totals = offline.simulate_pool(fx.pool, recs, ids, 4096, 0.4)
    assert len(metrics) == len(totals) == len(ids)
    for i, mid in enumerate(ids):
        model, pr, _, _ = fx.spec[mid]
        bank = offline.score_corpus(fx.banks[mid], recs, 'simulate', 4096, 0.4, divisor=32767)
        want_m, want_t = offline._metrics(fx.pool, recs, 4096, bank['above'][1].cpu().numpy(),
                                          bank['activations'][1].cpu().numpy(), bank['sum'][1].cpu().numpy())
        assert totals[i] == want_t, (mid, totals[i], want_t)
        assert metrics[i] == want_m
        assert metrics[i][0] is None
        one = m.PreciseB200(pr, hidden=model.hidden, activation=model.activation,
                            recurrent_activation=model.recurrent_activation)
        one.load_weights(model.kernel, model.recurrent, model.bias, model.dense_w, model.dense_b)
        _, t1 = offline.simulate(one, recs, 4096, 0.4)
        one.close()
        assert (t1.seconds, t1.activations, t1.activated_chunks) == (want_t.seconds, want_t.activations, want_t.activated_chunks)
        assert abs(t1.activation_sum - want_t.activation_sum) <= 1e-6 * max(1.0, abs(want_t.activation_sum))


def _write_folder(tmp_path):
    folder = tmp_path / 'noise'
    folder.mkdir()
    recs = {'a.wav': _noise(16000 * 20 + 5, 110), 'b.wav': _noise(40000, 111, 6000), 'c.wav': np.zeros(0, np.int16)}
    for name, a in recs.items():
        with wave.open(str(folder / name), 'wb') as w:
            w.setnchannels(1); w.setsampwidth(2); w.setframerate(16000); w.writeframes(a.tobytes())
    return folder


def _run_cli(args):
    """(rc, stdout without the loader's 'Warning:' lines about missing .params files, stderr)."""
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, '-m', 'mycroft_precise_b200.simulate'] + args, capture_output=True, env=env,
                       timeout=600)
    out = ''.join(line for line in r.stdout.decode().splitlines(True) if not line.startswith('Warning:'))
    return r.returncode, out, r.stderr.decode()


@gpu
def test_command_line_many_models(tmp_path):
    """Two and three .npz models: a heading per model, then exactly the blocks the one-model command prints for it."""
    m = _mod()
    folder = _write_folder(tmp_path)
    paths = []
    for i, (h, act) in enumerate([(20, 'linear'), (12, 'tanh'), (24, 'linear')]):
        g = m.GruModel.random(13, h, seed=40 + i, scale=0.3)
        if act == 'tanh':
            g.activation, g.recurrent_activation = 'tanh', 'sigmoid'
        p = str(tmp_path / ('model%d.npz' % i))
        m.save_weights(p, g)
        paths.append(p)
    single = []
    for p in paths:
        rc, out, err = _run_cli([p, str(folder), '-c', '4096', '-t', '0.3'])
        assert rc == 0, err[-2000:]
        assert '=== %s ===' % p not in out
        single.append(out)
    for n in (2, 3):
        rc, out, err = _run_cli(paths[:n] + [str(folder), '-c', '4096', '-t', '0.3'])
        assert rc == 0, err[-2000:]
        want = ''.join('\n=== %s ===\n' % p + s for p, s in zip(paths[:n], single[:n]))
        assert out == want
        assert len(re.findall(r'=== Total ===', out)) == n


def test_command_line_arguments(tmp_path, monkeypatch):
    """Without a device: several models parse before the folder; models that cannot share a pool are refused by name."""
    from mycroft_precise_b200 import simulate
    from mycroft_precise_b200.params import ListenerParams
    m = _mod()
    seen = {}

    def fake_resolve(path):
        seen.setdefault('paths', []).append(path)
        if path.endswith('wide.npz'):
            return m.GruModel.random(13, 32, seed=1), None
        if path.endswith('other.npz'):
            return m.GruModel.random(13, 20, seed=1), ListenerParams(hop_t=0.02)
        raise RuntimeError('stop after the checks')

    import mycroft_precise_b200.runner as runner
    monkeypatch.setattr(runner, '_resolve_model', fake_resolve)
    with pytest.raises(RuntimeError, match='stop after'):
        simulate.main(['a.npz', 'b.npz', 'folder'])
    assert seen['paths'] == ['a.npz']
    models = [(m.GruModel.random(13, 20, seed=0), ListenerParams())]
    with pytest.raises(ValueError, match='wide.npz'):
        simulate.check_pool_models(['a.npz', 'wide.npz'], models + [(m.GruModel.random(13, 32, seed=1), ListenerParams())])
    with pytest.raises(ValueError, match='other.npz.*hop_samples'):
        simulate.check_pool_models(['a.npz', 'other.npz'],
                                   models + [(m.GruModel.random(13, 20, seed=1), ListenerParams(hop_t=0.02))])
    with pytest.raises(ValueError, match='delta.npz'):
        simulate.check_pool_models(['delta.npz', 'a.npz'], [(m.GruModel.random(26, 20, seed=1), ListenerParams(use_delta=True)),
                                                            (m.GruModel.random(26, 20, seed=2), ListenerParams(use_delta=True))])
    simulate.check_pool_models(['a.npz', 'b.npz'], models * 2)
    with pytest.raises(SystemExit):
        simulate.main(['folder_only'])
