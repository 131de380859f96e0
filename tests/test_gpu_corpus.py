"""-m gpu: recorded corpora (pb_score_corpus, offline.score_corpus / simulate / false_activations, the precise-simulate
command line) against the oracle, the stateless path and the stream tick."""
import os
import re
import subprocess
import sys
import wave

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip('torch')

from oracle import gru as og              # noqa: E402
from oracle import mfcc as om             # noqa: E402
from oracle.decoder import OracleDecoder  # noqa: E402
from oracle.listener import OracleListener   # noqa: E402
from oracle.params import OracleParams    # noqa: E402
from oracle.trigger import OracleTrigger  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LENGTHS = [0, 1, 1599, 1600, 24800, 24801, 3333, 16000 * 20 + 5]


def _m():
    import mycroft_precise_b200 as m
    return m


def _noise(n, seed):
    rs = np.random.RandomState(seed)
    a = np.clip(rs.randn(n) * 3000 * (1 + np.sin(np.arange(n) / 4000.0)), -32768, 32767).astype(np.int16)
    if n > 8000:
        a[2000:6000] = 0
        a[6000:6500] = 32767
    return a


def _weights(model):
    return og.GruWeights(model.kernel, model.recurrent, model.bias, model.dense_w, model.dense_b,
                         activation=model.activation, recurrent_activation=model.recurrent_activation)


def _step(pr=None):
    p = OracleParams(**(pr.to_dict() if pr is not None else {}))
    d = OracleDecoder(p.threshold_config, p.threshold_center)
    return float(np.max(np.abs(np.diff(d.cd)))) * 2.5


def _oracle_listener(model, a, c, divisor, pr=None, sensitivity=0.5, trigger_level=3):
    """A fresh Listener + TriggerDetector of chunk c over one recording: (raw, conf, fired) per complete chunk."""
    opr = OracleParams(**(pr.to_dict() if pr is not None else {}))
    lis = OracleListener(_weights(model), opr)
    det = OracleTrigger(2 * c, sensitivity, trigger_level)
    K = len(a) // c
    raw, conf, fired = np.zeros(K, np.float32), np.zeros(K), np.zeros(K, bool)
    for k in range(K):
        r = lis.update_raw(a[k * c:(k + 1) * c].astype(np.float32) / np.float32(divisor))
        raw[k], conf[k] = r, lis.decoder.decode(r)
        fired[k] = det.update(conf[k])
    return raw, conf, fired


def _check_listener(got, wo, m_idx, recs, model, c, divisor, pr=None, sensitivity=0.5, trigger_level=3):
    """raw within 1e-4 of the oracle everywhere; fired equal up to the first window whose conf lies within one LUT bin of the
    hot threshold (after it the detectors may part); activations equal for every recording without such a window.  Returns
    how many recordings with windows were checked in full."""
    step = _step(pr)
    hot = 1.0 - sensitivity
    full = 0
    for i, a in enumerate(recs):
        raw, conf, fired = _oracle_listener(model, a, c, divisor, pr, sensitivity, trigger_level)
        sl = slice(wo[i], wo[i + 1])
        g_raw = got['raw'][m_idx, sl].cpu().numpy()
        g_fired = got['fired'][m_idx, sl].cpu().numpy().astype(bool)
        acts = int(got['activations'][m_idx, i])
        assert g_raw.shape == raw.shape, (i, c)
        if raw.size:
            assert np.max(np.abs(g_raw - raw)) < 1e-4, (i, c)
        near = np.abs(conf - hot) <= step
        first = int(np.argmax(near)) if near.any() else len(conf)
        assert np.array_equal(g_fired[:first], fired[:first]), (i, c)
        if first == len(conf):
            assert acts == int(fired.sum()), (i, c)
            full += raw.size > 0
        assert acts == int(g_fired.sum())
    return full


@pytest.mark.parametrize('c', [333, 800, 1024, 4000])
def test_listener_vs_oracle(c):
    m = _m()
    from mycroft_precise_b200 import offline
    model = m.GruModel.random(13, 20, seed=1, scale=0.1)
    core = m.PreciseB200()
    core.load_weights(model.kernel, model.recurrent, model.bias, model.dense_w, model.dense_b)
    recs = [_noise(L, 10 + i) for i, L in enumerate(LENGTHS)]
    for divisor in ((32768, 32767) if c == 1024 else (32768,)):
        got = offline.score_corpus(core, recs, 'listener', c, divisor=divisor)
        wo = got['window_offsets']
        assert list(np.diff(wo)) == [L // c for L in LENGTHS]
        assert got['above'] is None and got['sum'] is None
        assert _check_listener(got, wo, 0, recs, model, c, divisor) >= 3
    core.close()


def test_listener_bank_delta_wide():
    m = _m()
    from mycroft_precise_b200 import offline
    c = 1024
    recs = [_noise(L, 30 + i) for i, L in enumerate([0, 24801, 16000 * 20 + 5, 5000])]
    m0 = m.GruModel.random(13, 20, seed=0, scale=0.1)
    m1 = m.GruModel.random(13, 20, seed=2, scale=0.1)
    m1.activation, m1.recurrent_activation = 'tanh', 'sigmoid'
    m2 = m.GruModel.random(13, 128, seed=3, scale=0.1 / np.sqrt(128 / 20.0))
    core = m.PreciseB200(sensitivity=0.8, trigger_level=1)
    core.load_weights(m0.kernel, m0.recurrent, m0.bias, m0.dense_w, m0.dense_b)
    core.add_model(m1, sensitivity=0.5, trigger_level=3)
    core.add_model(m2, sensitivity=0.5, trigger_level=2)
    got = offline.score_corpus(core, recs, 'listener', c)
    for i, (model, sens, lvl) in enumerate([(m0, 0.8, 1), (m1, 0.5, 3), (m2, 0.5, 2)]):
        assert _check_listener(got, got['window_offsets'], i, recs, model, c, 32768, None, sens, lvl) >= 1
    core.close()
    pr = m.ListenerParams(use_delta=True)
    md = m.GruModel.random(26, 20, seed=4, scale=0.1)
    core = m.PreciseB200(pr, sensitivity=0.8, trigger_level=1)
    core.load_weights(md.kernel, md.recurrent, md.bias, md.dense_w, md.dense_b)
    got = offline.score_corpus(core, recs, 'listener', c)
    assert _check_listener(got, got['window_offsets'], 0, recs, md, c, 32768, pr, 0.8, 1) >= 1
    core.close()


def test_listener_vs_stream_ticks():
    """Each recording one stream of StreamBatch, one tick per chunk; and one recording of 10 minutes (> 8 192 windows: the
    large-batch scan) against a single stream."""
    m = _m()
    from mycroft_precise_b200 import offline
    model = m.GruModel.random(13, 20, seed=5, scale=0.1)
    c, K, S = 1024, 40, 5
    recs = [_noise(K * c, 50 + s) for s in range(S)]
    core = m.PreciseB200()
    core.load_weights(model.kernel, model.recurrent, model.bias, model.dense_w, model.dense_b)
    got = offline.score_corpus(core, recs, 'listener', c)
    sb = m.StreamBatch(model, S, chunk_samples=c)
    pcm = np.stack(recs)
    raw, conf, fired = np.zeros((S, K), np.float32), np.zeros((S, K)), np.zeros((S, K), bool)
    for k in range(K):
        o = sb.update(torch.from_numpy(pcm[:, k * c:(k + 1) * c].copy()).cuda())
        raw[:, k], conf[:, k], fired[:, k] = o['raw'].cpu().numpy(), o['conf'].cpu().numpy(), o['fired'].cpu().numpy() > 0
    step = _step()
    g_raw = got['raw'][0].cpu().numpy().reshape(S, K)
    g_fired = got['fired'][0].cpu().numpy().reshape(S, K) > 0
    assert np.max(np.abs(g_raw - raw)) < 1e-5
    acts = got['activations'][0].cpu().numpy()
    near = np.abs(conf - 0.5) <= step
    for s_ in range(S):
        first = int(np.argmax(near[s_])) if near[s_].any() else K
        assert np.array_equal(g_fired[s_, :first], fired[s_, :first]), s_
        assert acts[s_] == int(g_fired[s_].sum())
        if first == K:
            assert acts[s_] == int(fired[s_].sum()), s_
    # 10 minutes, one stream
    long = _noise(16000 * 600, 60)
    K = len(long) // c
    got = offline.score_corpus(core, [long], 'listener', c)
    assert got['raw'].shape[1] == K > 8192
    sb1 = m.StreamBatch(model, 1, chunk_samples=c)
    dev = torch.from_numpy(long[:K * c].reshape(K, 1, c).copy()).cuda()
    raw1 = torch.empty(K, dtype=torch.float32, device='cuda')
    for k in range(K):
        raw1[k] = sb1.update(dev[k])['raw'][0]
    assert float((got['raw'][0] - raw1).abs().max()) < 1e-5
    core.close()


def _simulate_oracle(model, a, chunk, threshold, pr=None, divisor=32767):
    """SimulateScript.run's numbers for one recording (simulate.py:92-120), oracle MFCC and network, load_audio scaling."""
    from mycroft_precise_b200.runner import TriggerDetector
    opr = OracleParams(**(pr.to_dict() if pr is not None else {}))
    if len(a) < opr.window_samples:
        return np.zeros(0, np.float32), 0, 0, 0.0
    mf = om.vectorize_raw(a.astype(np.float32) / np.float32(divisor), opr)
    hops = chunk // opr.hop_samples
    ends = range(opr.n_features, len(mf), hops)
    if len(ends) == 0:
        return np.zeros(0, np.float32), 0, 0, 0.0
    pred = og.predict(_weights(model), np.array([mf[i - opr.n_features:i] for i in ends]))
    det = TriggerDetector(chunk, trigger_level=0, sensitivity=threshold)
    return pred[:, 0], int((pred > threshold).sum()), int(sum(det.update(p) for p in pred)), float(pred.sum())


def test_simulate_vs_evaluate_and_oracle():
    m = _m()
    from mycroft_precise_b200 import offline
    model = m.GruModel.random(13, 20, seed=6, scale=0.3)
    core = m.PreciseB200()
    core.load_weights(model.kernel, model.recurrent, model.bias, model.dense_w, model.dense_b)
    lens = [0, 1, 24000, 24800, 25600, 24801, 16000 * 20, 16000 * 20 + 5]
    recs = [_noise(L, 70 + i) for i, L in enumerate(lens)]
    for chunk in (1600, 4096):
        got = offline.score_corpus(core, recs, 'simulate', chunk, 0.5, divisor=32768)
        wo = got['window_offsets']
        for i, a in enumerate(recs):
            g = got['raw'][0, wo[i]:wo[i + 1]]
            if len(a) == 0:
                assert g.numel() == 0
                continue
            want = offline.evaluate(core, a, chunk)           # its chunk_size // hop_samples, as simulate.py:96
            assert g.shape == want.shape
            if g.numel() and len(a) % 8 == 0:                             # same MFCC kernel, same network kernel
                assert torch.equal(g, want), (i, chunk)
            if g.numel():
                assert float((g - want).abs().max()) < 1e-5
    for thr in (0.5, 0.2):
        metrics, total = offline.simulate(core, recs, 4096, thr)
        assert metrics[0] is None
        tot = [0, 0, 0.0]
        for i, a in enumerate(recs[1:], 1):
            pred, above, acts, s = _simulate_oracle(model, a, 4096, thr)
            mt = metrics[i]
            assert mt.seconds == len(a) / 16000.0
            near = np.abs(pred - thr) < 1e-5
            if not near.any():
                assert mt.activated_chunks == above and mt.activations == acts, (i, thr)
            assert abs(mt.activation_sum - s) <= 1e-4 * max(1.0, abs(s))
            tot[0] += mt.activated_chunks; tot[1] += mt.activations; tot[2] += mt.activation_sum
        assert (total.activated_chunks, total.activations) == (tot[0], tot[1])
    core.close()


def test_corpus_calls_leave_streams_alone():
    m = _m()
    from mycroft_precise_b200 import offline
    model = m.GruModel.random(13, 20, seed=7, scale=0.1)
    S, c, K = 9, 1024, 12
    pcm = np.stack([_noise(K * c, 80 + s) for s in range(S)])
    a, b = m.StreamBatch(model, S, chunk_samples=c), m.StreamBatch(model, S, chunk_samples=c)
    recs = [_noise(L, 90 + i) for i, L in enumerate(LENGTHS)]
    side = torch.cuda.Stream()
    for k in range(K):
        x = torch.from_numpy(pcm[:, k * c:(k + 1) * c].copy()).cuda()
        oa, ob = a.update(x), b.update(x)
        for key in ('raw', 'conf', 'fired'):
            assert torch.equal(oa[key], ob[key])
        if k % 3 == 0:
            offline.score_corpus(a.core, recs, 'listener', 333)
        if k % 3 == 1:
            with torch.cuda.stream(side):
                offline.score_corpus(a.core, recs, 'simulate', 4096)
    torch.cuda.synchronize()
    assert torch.equal(a.core.export_streams(), b.core.export_streams())


def test_false_activations_vs_oracle():
    m = _m()
    from mycroft_precise_b200 import offline
    model = m.GruModel.random(13, 20, seed=8, scale=0.3)
    core = m.PreciseB200()
    core.load_weights(model.kernel, model.recurrent, model.bias, model.dense_w, model.dense_b)
    c = 2048
    recs = [_noise(L, 100 + i) for i, L in enumerate([0, 2048, 2049, 30000, 16000 * 20 + 5])]
    thr = 0.4
    got = offline.false_activations(core, recs, c, thr)
    step = _step()
    bs = m.ListenerParams().buffer_samples
    want, near = {}, set()
    for i, a in enumerate(recs):
        audio = a.astype(np.float32) / np.float32(32767)
        lis = OracleListener(_weights(model), OracleParams())
        buf = np.zeros(bs, np.float32)
        for k, st in enumerate(range(c, len(audio), c)):                 # chunk_audio (util.py:30-32)
            chunk = audio[st - c:st]
            buf = np.concatenate((buf[len(chunk):], chunk))
            conf = lis.update(chunk)
            if abs(conf - thr) <= step:
                near.add((i, k))
            if conf > thr:
                want[(i, k)] = buf.copy()
    gotd = {(i, k): clip for i, k, clip in got}
    assert set(gotd) - near == set(want) - near
    assert len(want) > 0
    for key in set(gotd) & set(want):
        assert np.array_equal(gotd[key], want[key]), key
    core.close()


def test_simulate_command_line(tmp_path):
    m = _m()
    from mycroft_precise_b200.offline import Metric
    model = m.GruModel.random(13, 20, seed=9, scale=0.3)
    path = str(tmp_path / 'model.npz')
    m.save_weights(path, model)
    folder = tmp_path / 'noise'
    folder.mkdir()
    recs = {'a.wav': _noise(16000 * 20 + 5, 110), 'b.wav': _noise(40000, 111), 'c.wav': _noise(0, 112)}
    for name, a in recs.items():
        with wave.open(str(folder / name), 'wb') as w:
            w.setnchannels(1); w.setsampwidth(2); w.setframerate(16000); w.writeframes(a.tobytes())
    (folder / 'd.wav').write_bytes(b'not a wav file')
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, '-m', 'mycroft_precise_b200.simulate', path, str(folder), '-c', '4096', '-t', '0.3'],
                       capture_output=True, env=env, timeout=600)
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    out = r.stdout.decode()
    blocks = re.findall(r'=== (\S+) ===\nHours: (\S+)\nActivations / Day: (\S+)\nActivated Chunks / Day: (\S+)\n'
                        r'Average Activation \(\*100\): (\S+)', out)
    assert sorted(b[0] for b in blocks) == ['Total', 'a.wav', 'b.wav']
    total = Metric(4096)
    for name in ('a.wav', 'b.wav'):
        pred, above, acts, s = _simulate_oracle(model, recs[name], 4096, 0.3)
        mt = Metric(4096, len(recs[name]) / 16000.0, above, acts, s)
        total.add(mt)
        want = mt.info_string(name)
        got = [b for b in blocks if b[0] == name][0]
        want_nums = re.findall(r': (\S+)', want)
        for g, w in zip(got[1:], want_nums):
            assert abs(float(g) - float(w)) <= 0.011 + 1e-4 * abs(float(w)), (name, got, want)
    assert blocks[-1][0] == 'Total'
    want_nums = re.findall(r': (\S+)', total.info_string('Total'))
    for g, w in zip(blocks[-1][1:], want_nums):
        assert abs(float(g) - float(w)) <= 0.011 + 1e-4 * abs(float(w)), (blocks[-1], want_nums)


@pytest.mark.parametrize('mode', ['unaligned', 'force_generic', 'n_fft256', 'speechpy'])
def test_generic_k1_both_schedules(mode):
    """The generic corpus K1 (mfcc_corpus_kernel): recordings packed back to back from offset 1 (offsets 1, 2 and 7 mod 8),
    on the default handle, with force_generic, n_fft 256 and the speechpy vectoriser (release window + hop).  Listener
    against oracle Listeners; simulate raw bit for bit against offline.evaluate with pb_mfcc on its generic kernel (the same
    per-frame code and, at one model and <= 8 192 windows, the same network kernel), and within 1e-4 of the oracle."""
    m = _m()
    from mycroft_precise_b200 import offline
    pr = {'unaligned': m.ListenerParams(), 'force_generic': m.ListenerParams(), 'n_fft256': m.ListenerParams(n_fft=256),
          'speechpy': m.ListenerParams(vectorizer=3)}[mode]
    model = m.GruModel.random(pr.feature_size, 20, seed=11, scale=0.1)
    core = m.PreciseB200(pr, sensitivity=0.8, trigger_level=1)
    core.load_weights(model.kernel, model.recurrent, model.bias, model.dense_w, model.dense_b)
    if mode == 'force_generic':
        core.force_generic(True)
    lens = [0, 1, 1599, 1600, 24801, 33333, 16000 * 8 + 3]
    recs = [_noise(L, 120 + i) for i, L in enumerate(lens)]
    offs = np.concatenate([[1], 1 + np.cumsum(lens)]).astype(np.int64)
    assert sorted({int(o) % 8 for o, L in zip(offs[:-1], lens) if L}) == [1, 2, 7]
    host = np.zeros(int(offs[-1]), np.int16)
    for a, o in zip(recs, offs[:-1]):
        host[o:o + len(a)] = a
    pcm = torch.from_numpy(host).cuda()
    for c in (333, 1024):
        got = core.score_corpus(pcm, offs, 'listener', c)
        wo = np.concatenate([[0], np.cumsum([core.corpus_windows(L, 'listener', c) for L in lens])])
        assert wo[-1] == got['raw'].shape[1]
        assert _check_listener(got, wo, 0, recs, model, c, 32768, pr, 0.8, 1) >= 2
    chunk = 1600
    got = core.score_corpus(pcm, offs, 'simulate', chunk, 0.5)
    wo = np.concatenate([[0], np.cumsum([core.corpus_windows(L, 'simulate', chunk) for L in lens])])
    assert wo[-1] == got['raw'].shape[1] and wo[-1] > 50
    core.force_generic(True)
    checked = 0
    for i, a in enumerate(recs):
        g = got['raw'][0, wo[i]:wo[i + 1]]
        if len(a) < pr.window_samples:
            assert g.numel() == 0
            continue
        want = offline.evaluate(core, a, chunk)
        assert g.shape == want.shape, i
        if g.numel():
            assert torch.equal(g, want), (mode, i)
            pred, above, acts, s = _simulate_oracle(model, a, chunk, 0.5, pr, 32768)
            assert np.max(np.abs(g.cpu().numpy() - pred)) < 1e-4
            checked += 1
    assert checked >= 2
    core.close()
