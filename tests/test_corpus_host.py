"""Recorded corpora without a device: window counts of pb_corpus_windows, argument errors, the wav reader of the
precise-simulate command line and the Metric arithmetic and format (precise/scripts/simulate.py:45-80)."""
import ctypes as C
import wave

import numpy as np
import pytest

from mycroft_precise_b200.core import get_lib, make_config
from mycroft_precise_b200.offline import Metric
from mycroft_precise_b200.params import ListenerParams
from mycroft_precise_b200.simulate import InvalidAudio, read_wav


def _frames(pr, n):
    rel = pr.window_samples + (pr.hop_samples if pr.vectorizer == 3 else 0)
    return 0 if n < rel else (n - rel) // pr.hop_samples + 1


@pytest.mark.parametrize('vectorizer', [2, 3])
def test_corpus_windows_match_reference_formulas(vectorizer):
    lib = get_lib()
    pr = ListenerParams(vectorizer=vectorizer)
    cfg = make_config(pr)
    win = pr.window_samples
    lengths = [0, 1, win - 1, win, win + 1, 1601, 24799, 24800, 24801, 33333, 16000 * 20 + 7]
    for n in lengths:
        nf = _frames(pr, n)
        for c in (800, 1600, 4096, 4097, 8000):
            assert lib.pb_corpus_windows(C.byref(cfg), 1, c, n) == len(range(pr.n_features, nf, c // pr.hop_samples)), (n, c)
        for c in (1, 333, 1024, 4000):
            assert lib.pb_corpus_windows(C.byref(cfg), 0, c, n) == n // c, (n, c)


def test_corpus_argument_errors():
    lib = get_lib()
    cfg = make_config(ListenerParams())
    assert lib.pb_corpus_windows(None, 0, 1024, 10) == -1
    assert lib.pb_corpus_windows(C.byref(cfg), 2, 1024, 10) == -1          # unknown schedule
    assert lib.pb_corpus_windows(C.byref(cfg), 0, 0, 10) == -1             # chunk < 1
    assert lib.pb_corpus_windows(C.byref(cfg), 1, 799, 10) == -1           # simulate: chunk // hop = 0
    assert lib.pb_corpus_windows(C.byref(cfg), 0, 1024, -1) == -1
    offs = np.zeros(2, np.int64)
    raw = C.c_void_p(8)
    assert lib.pb_score_corpus(None, None, offs.ctypes.data_as(C.c_void_p), 1, 32768, 0, 1024, 0.5, raw,
                               None, None, None, None, None, None) == -1


def _write(path, data, width=2, rate=16000, channels=1):
    with wave.open(str(path), 'wb') as w:
        w.setnchannels(channels)
        w.setsampwidth(width)
        w.setframerate(rate)
        w.writeframes(data)


def test_wav_reader(tmp_path):
    a = (np.arange(1000) * 37 % 65536 - 32768).astype(np.int16)
    _write(tmp_path / 'ok.wav', a.tobytes())
    assert np.array_equal(read_wav(str(tmp_path / 'ok.wav')), a)
    _write(tmp_path / 'empty.wav', b'')
    assert read_wav(str(tmp_path / 'empty.wav')).size == 0
    (tmp_path / 'broken.wav').write_bytes(b'RIFF\x10\x00\x00\x00WAVEjunk')
    assert read_wav(str(tmp_path / 'broken.wav')).size == 0
    (tmp_path / 'zero.wav').write_bytes(b'')
    assert read_wav(str(tmp_path / 'zero.wav')).size == 0
    _write(tmp_path / 'u8.wav', bytes(100), width=1)
    with pytest.raises(InvalidAudio):
        read_wav(str(tmp_path / 'u8.wav'))
    _write(tmp_path / 'rate.wav', a.tobytes(), rate=44100)
    with pytest.raises(InvalidAudio):
        read_wav(str(tmp_path / 'rate.wav'))
    _write(tmp_path / 'stereo.wav', a.tobytes(), channels=2)
    with pytest.raises(InvalidAudio):
        read_wav(str(tmp_path / 'stereo.wav'))


def test_metric_arithmetic_and_format():
    m = Metric(4096, seconds=7200.0, activated_chunks=12, activations=3, activation_sum=25.5)
    assert m.days == pytest.approx(7200.0 / 86400)
    assert m.chunks == pytest.approx(7200.0 * 16000 / 4096)
    t = Metric(4096)
    t.add(m)
    t.add(Metric(4096, 3600.0, 1, 1, 0.5))
    assert (t.seconds, t.activated_chunks, t.activations, t.activation_sum) == (10800.0, 13, 4, 26.0)
    days = 7200.0 / 86400
    want = ('=== f.wav ===\n'
            'Hours: %.2f\n'
            'Activations / Day: %.2f\n'
            'Activated Chunks / Day: %.2f\n'
            'Average Activation (*100): %.2f') % (days * 24, 3 / days, 12 / days, 100.0 * 25.5 / (7200.0 * 16000 / 4096))
    assert m.info_string('f.wav') == want
