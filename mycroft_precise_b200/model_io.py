"""Model weights for the GRU + Dense network (precise/model.py:77-82).

Native format: ``<name>.npz`` with keys kernel[F,3H], recurrent[H,3H], bias[3H], dense_w[H],
dense_b, plus optional activation / recurrent_activation strings, next to the reference's own
``<name>.params`` JSON (precise/params.py:150-165).  Keras gate order z, r, h.
"""
import numpy as np

MODEL_SUFFIXES = ('.npz', '.pb', '.net')      # own format, frozen GraphDef, Keras HDF5 (Listener.find_runner: network_runner.py:111-119)


class GruModel:
    def __init__(self, kernel, recurrent, bias, dense_w, dense_b, activation='linear',
                 recurrent_activation='hard_sigmoid'):
        self.kernel = np.ascontiguousarray(kernel, dtype=np.float32)
        self.recurrent = np.ascontiguousarray(recurrent, dtype=np.float32)
        self.bias = np.ascontiguousarray(bias, dtype=np.float32).reshape(-1)
        self.dense_w = np.ascontiguousarray(dense_w, dtype=np.float32).reshape(-1)
        self.dense_b = float(np.asarray(dense_b, dtype=np.float32).reshape(-1)[0])
        self.activation = str(activation)
        self.recurrent_activation = str(recurrent_activation)
        self.hidden = self.recurrent.shape[0]
        self.feature_size = self.kernel.shape[0]
        H = self.hidden
        if (self.kernel.shape[1] != 3 * H or self.recurrent.shape != (H, 3 * H) or
                self.bias.shape != (3 * H,) or self.dense_w.shape != (H,)):
            raise ValueError('inconsistent GRU weight shapes')

    @staticmethod
    def random(feature_size=13, hidden=20, seed=0, scale=0.3):
        """Seeded synthetic weights (the reference ships no trained model)."""
        rs = np.random.RandomState(seed)
        return GruModel(rs.randn(feature_size, 3 * hidden) * scale, rs.randn(hidden, 3 * hidden) * scale,
                        rs.randn(3 * hidden) * scale, rs.randn(hidden) * scale, rs.randn(1) * scale)

    @staticmethod
    def init(feature_size=13, hidden=20, seed=0, activation='linear', recurrent_activation='hard_sigmoid'):
        """A new network as Keras initialises GRU and Dense layers, from numpy's RandomState(seed): glorot_uniform kernel
        and dense weights (uniform in +-sqrt(6 / (fan_in + fan_out))), an orthogonal recurrent kernel [H, 3H] (the Q factor
        of a standard normal matrix, as keras.initializers.Orthogonal builds it) and zero biases."""
        rs = np.random.RandomState(seed)
        F, H = feature_size, hidden
        lim = np.sqrt(6.0 / (F + 3 * H))
        kernel = rs.uniform(-lim, lim, (F, 3 * H))
        a = rs.normal(0.0, 1.0, (H, 3 * H))
        u, _, v = np.linalg.svd(a, full_matrices=False)
        recurrent = u if u.shape == (H, 3 * H) else v
        lim_d = np.sqrt(6.0 / (H + 1))
        dense_w = rs.uniform(-lim_d, lim_d, H)
        return GruModel(kernel, recurrent, np.zeros(3 * H), dense_w, 0.0, activation, recurrent_activation)


def save_weights(path: str, m: GruModel):
    np.savez(path, kernel=m.kernel, recurrent=m.recurrent, bias=m.bias, dense_w=m.dense_w,
             dense_b=np.float32(m.dense_b), activation=m.activation,
             recurrent_activation=m.recurrent_activation)


def load_weights(path: str) -> GruModel:
    if path.endswith('.npz'):
        z = np.load(path, allow_pickle=False)
        return GruModel(z['kernel'], z['recurrent'], z['bias'], z['dense_w'], z['dense_b'],
                        str(z['activation']) if 'activation' in z else 'linear',
                        str(z['recurrent_activation']) if 'recurrent_activation' in z else 'hard_sigmoid')
    if path.endswith('.pb'):
        from .pb_import import load_pb
        return load_pb(path)
    if path.endswith('.net'):
        return load_net(path)
    raise ValueError('File extension of ' + path + " must be: ['.npz', '.pb', '.net']")


def _as_str(v):
    if isinstance(v, bytes):
        return v.decode('utf-8')
    if isinstance(v, np.ndarray) and v.shape == ():
        return _as_str(v.item())
    return str(v)


def model_from_keras_h5(f) -> GruModel:
    """Weights of the reference network from an open Keras HDF5 model file (``create_model``, precise/model.py:72-82:
    ``GRU(units, name='net', activation='linear', ...)`` then ``Dense(1, activation='sigmoid')``; what ``model.save`` wrote,
    precise/model.py:55-57 / scripts/train.py).  ``f`` is an ``h5py.File`` or anything with the same mapping interface:
    ``f.attrs['model_config']`` (JSON) and ``f['model_weights'][layer][<weight names>]`` (``model_weights`` is absent in
    weight-only files, where the layer groups sit at the root)."""
    import json
    root = f['model_weights'] if 'model_weights' in f else f
    act, ract = 'linear', 'hard_sigmoid'
    gru_name, dense_name = 'net', None
    if 'model_config' in f.attrs:
        cfg = json.loads(_as_str(f.attrs['model_config']))
        layers = cfg.get('config', cfg)
        layers = layers.get('layers', layers) if isinstance(layers, dict) else layers
        for ly in layers:
            c = ly.get('config', {})
            if ly.get('class_name') == 'GRU':
                gru_name = c.get('name', gru_name)
                act = c.get('activation', act)
                ract = c.get('recurrent_activation', ract)
                if c.get('reset_after', False):
                    raise ValueError('GRU(reset_after=True) is not the reference network (precise/model.py:77-80)')
            elif ly.get('class_name') == 'Dense':
                dense_name = c.get('name', dense_name)
                if c.get('activation', 'sigmoid') != 'sigmoid':
                    raise ValueError('the output layer must be Dense(1, activation="sigmoid")')

    def datasets(group):
        out = {}

        def walk(g, prefix):
            for k in g.keys():
                v = g[k]
                if hasattr(v, 'keys'):
                    walk(v, prefix + k + '/')
                else:
                    out[prefix + k] = np.asarray(v)
        walk(group, '')
        return out

    if dense_name is None:
        cands = [k for k in root.keys() if k.startswith('dense')]
        if len(cands) != 1:
            raise ValueError('cannot identify the Dense layer among %r' % list(root.keys()))
        dense_name = cands[0]
    g = datasets(root[gru_name])
    d = datasets(root[dense_name])

    def pick(ds, stem):
        hits = [v for k, v in ds.items() if k.split('/')[-1].split(':')[0] == stem]
        if len(hits) != 1:
            raise ValueError('expected one %r among %r' % (stem, sorted(ds)))
        return hits[0]
    k, u, b, dw, db = pick(g, 'kernel'), pick(g, 'recurrent_kernel'), pick(g, 'bias'), pick(d, 'kernel'), pick(d, 'bias')
    # strict shape / dtype check: a mis-parsed file must not load plausible-looking garbage
    H = u.shape[0] if u.ndim == 2 else -1
    ok = (k.ndim == 2 and u.ndim == 2 and k.shape[1] == 3 * H and u.shape == (H, 3 * H) and b.shape == (3 * H,)
          and dw.shape in ((H, 1), (H,)) and db.shape in ((1,), ()))
    if not ok or any(a.dtype.kind != 'f' for a in (k, u, b, dw, db)):
        raise ValueError('unexpected GRU / Dense dataset shapes or types in the Keras file: kernel %s %s, recurrent_kernel %s %s, '
                         'bias %s %s, dense kernel %s %s, dense bias %s %s' % (k.shape, k.dtype, u.shape, u.dtype, b.shape, b.dtype,
                                                                              dw.shape, dw.dtype, db.shape, db.dtype))
    return GruModel(k, u, b, dw.reshape(-1), db, act, ract)


def load_net(path: str) -> GruModel:
    """Keras ``.net`` (HDF5) model file: through ``h5py`` where it is installed (wherever the reference itself runs -- Keras
    depends on it), otherwise through the built-in reader for h5py's default file format (``h5_import.py``; written from the
    HDF5 specification, not validated against Keras-written files in this build image).  A file the built-in reader refuses
    (``libver='latest'``, compression) can be converted where h5py exists:
    ``python -m mycroft_precise_b200.model_io model.net model.npz``."""
    try:
        import h5py
    except ImportError:
        import warnings
        from .h5_import import H5File
        warnings.warn('h5py is not installed: reading %s with the built-in HDF5 reader (validated against spec-following test files '
                      'only, not against Keras-written files); convert once where h5py exists if in doubt' % path, RuntimeWarning)
        with H5File(path) as f:
            return model_from_keras_h5(f)
    with h5py.File(path, 'r') as f:
        return model_from_keras_h5(f)


if __name__ == '__main__':
    import shutil
    import sys
    if len(sys.argv) != 3:
        sys.exit('usage: python -m mycroft_precise_b200.model_io <model.net|model.pb|model.npz> <out.npz>')
    save_weights(sys.argv[2], load_weights(sys.argv[1]))
    import os
    if os.path.isfile(sys.argv[1] + '.params'):
        shutil.copyfile(sys.argv[1] + '.params', sys.argv[2] + '.params')
    print('wrote', sys.argv[2])
