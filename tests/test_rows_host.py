"""CPU-only: the test command's choice between the pool path (offline.test_pool) and the weight-row path (offline.test_rows),
its refusals before any device work, and TrainState.from_models' packing of a wide set read back by models()."""
import numpy as np
import pytest

import mycroft_precise_b200 as m
from mycroft_precise_b200 import core as mcore
from mycroft_precise_b200 import offline
from mycroft_precise_b200 import test as ptest
from mycroft_precise_b200.model_io import GruModel, save_weights
from mycroft_precise_b200.params import ListenerParams, save_params


class _Stop(Exception):
    pass


def _save(tmp_path, name, F, H, params=None, seed=0):
    path = str(tmp_path / name)
    save_weights(path, GruModel.random(F, H, seed=seed))
    save_params(path, params or ListenerParams())
    return path


@pytest.fixture
def calls(monkeypatch, tmp_path):
    """Stands in for the device: records which path the command takes and stops it there."""
    seen = []

    class Core:
        def __init__(self, *a, **kw):
            seen.append('core')

        def set_pool(self, n):
            pass

        def pool_load(self, *a):
            pass

    def path(name):
        def f(*a, **kw):
            seen.append(name)
            raise _Stop()
        return f

    monkeypatch.setattr(mcore, 'PreciseB200', Core)
    monkeypatch.setattr(offline, 'test_pool', path('test_pool'))
    monkeypatch.setattr(offline, 'vectorize_clips', path('test_rows'))
    (tmp_path / 'data' / 'test').mkdir(parents=True)
    return seen


def test_fused_sets_take_the_pool_and_wide_sets_the_rows(tmp_path, calls):
    data = str(tmp_path / 'data')
    a, b = _save(tmp_path, 'a.npz', 13, 20), _save(tmp_path, 'b.npz', 13, 24, seed=1)
    wide, top = _save(tmp_path, 'w.npz', 13, 25), _save(tmp_path, 't.npz', 13, 128)
    for models, want in (([a], 'test_pool'), ([a, b], 'test_pool'), ([wide], 'test_rows'), ([a, top], 'test_rows'),
                         ([top, wide, b], 'test_rows')):
        calls.clear()
        with pytest.raises(_Stop):
            ptest.main(models + [data])
        assert calls == ['core', want], models


def test_refusals_come_before_any_device_work(tmp_path, calls):
    data = str(tmp_path / 'data')
    wide = _save(tmp_path, 'w.npz', 13, 64)
    cases = [(_save(tmp_path, 'h129.npz', 13, 129), 'hidden <= 128'),
             (_save(tmp_path, 'mfcc16.npz', 16, 20, ListenerParams(n_mfcc=16)), 'front end differs'),
             (_save(tmp_path, 'delta.npz', 26, 64, ListenerParams(use_delta=True)), 'front end differs')]
    for bad, msg in cases:
        calls.clear()
        with pytest.raises(ValueError, match=msg):
            ptest.main([wide, bad, data])
        assert calls == []
    # the first model's own front end outside the row path's range: deltas, feature size 17
    for params, F in ((ListenerParams(use_delta=True), 26), (ListenerParams(n_filt=20, n_mfcc=17), 17)):
        bad = _save(tmp_path, 'first%d.npz' % F, F, 40, params)
        calls.clear()
        with pytest.raises(ValueError, match='feature size <= 16 and no deltas'):
            ptest.main([bad, data])
        assert calls == []
    # a fused set keeps the pool's own refusal
    calls.clear()
    with pytest.raises(ValueError, match='only networks of the fused family'):
        ptest.main([_save(tmp_path, 'f17.npz', 17, 20, ListenerParams(n_filt=20, n_mfcc=17)), data])
    assert calls == []


def test_from_models_packs_a_wide_set_that_models_reads_back():
    torch = pytest.importorskip('torch')

    class Core:
        feature_size = 13
        device = torch.device('cpu')
        train_rows = staticmethod(mcore.PreciseB200.train_rows)

    core = Core()
    core.torch = torch
    models = [GruModel.random(13, H, seed=H) for H in (1, 24, 25, 64, 128)]
    models[1].activation, models[1].recurrent_activation = 'tanh', 'sigmoid'
    st = offline.TrainState.from_models(core, models, [5, 6, 7, 8, 9])
    assert st.wide and st.stride == m.core.PB_TRAIN_WIDE_STRIDE and tuple(st.weights.shape) == (5, st.stride)
    w = st.weights.numpy()
    for i, (g, back) in enumerate(zip(models, st.models())):
        H = g.hidden
        n = 3 * H * (13 + H + 1) + H + 1
        assert not np.any(w[i, n:])
        for name in ('kernel', 'recurrent', 'bias', 'dense_w'):
            assert np.array_equal(getattr(back, name), getattr(g, name).astype(np.float32)), (H, name)
        assert np.float32(back.dense_b) == np.float32(g.dense_b)
        assert (back.activation, back.recurrent_activation) == (g.activation, g.recurrent_activation)
    assert [r.hidden for r in st.rows[0][:5]] == [1, 24, 25, 64, 128] and [r.seed for r in st.rows[0][:5]] == [5, 6, 7, 8, 9]
    fused = offline.TrainState.from_models(core, models[:2], [0, 1])
    assert not fused.wide and fused.stride == m.core.PB_TRAIN_STRIDE
