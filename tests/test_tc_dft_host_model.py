"""CPU: the tensor-core formulation of the MFCC DFT -- the 16-point real-DFT butterfly, the fp16 hi/lo operands of the 64 x 64
stage-2 matrix and the accumulator-column -> bin map (csrc/mfcc_tc.cuh, csrc/mfcc_tc3.cuh) -- reproduces a float64 power
spectrum, and so does the DFT of the mma.sync MFCC tick read through that kernel's own fragment tables (csrc/mfcc_mma.cuh).
The library exports these CPU models (pb_debug_tc_dft_power, pb_debug_mma_dft_power, ...); no device is needed."""
import ctypes as C

import numpy as np
import pytest

from mycroft_precise_b200.core import get_lib


def _power(x):
    lib = get_lib()
    x = np.ascontiguousarray(x, dtype=np.int16)
    out = np.zeros(257, np.float64)
    rc = lib.pb_debug_tc_dft_power(x.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
    assert rc == 0
    return out


def _cases():
    rs = np.random.RandomState(7)
    yield 'noise', np.clip(rs.randn(512) * 3000, -32768, 32767)
    yield 'quiet', np.round(rs.randn(512) * 2)
    yield 'max dc', np.full(512, 32767)
    yield 'min dc', np.full(512, -32768)
    yield 'nyquist', np.where(np.arange(512) % 2 == 0, 32767, -32768)
    yield 'impulse', np.eye(1, 512, 137).ravel() * 30000
    yield 'tone', 32000 * np.sin(2 * np.pi * 1000 / 16000 * np.arange(512) + 0.3)
    for k in (1, 7, 8, 9, 15, 16, 17, 100, 129, 255):                 # one bin from every GEMM block / column quarter
        yield 'bin %d' % k, 20000 * np.cos(2 * np.pi * k * np.arange(512) / 512 + 0.1 * k)


@pytest.mark.parametrize('name,x', list(_cases()), ids=[n for n, _ in _cases()])
def test_host_model_matches_float64_fft(name, x):
    x = np.asarray(x).astype(np.int16)
    ref = np.abs(np.fft.rfft(x.astype(np.float64))) ** 2
    got = _power(x)
    peak = max(ref.max(), 1.0)
    assert np.max(np.abs(got - ref)) / peak < 3e-6, name


def test_silence_is_exactly_zero():
    assert np.all(_power(np.zeros(512, np.int16)) == 0.0)


def _mma_power(x):
    lib = get_lib()
    x = np.ascontiguousarray(x, dtype=np.int16)
    out = np.zeros(257, np.float64)
    assert lib.pb_debug_mma_dft_power(x.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)) == 0
    return out


@pytest.mark.parametrize('name,x', list(_cases()), ids=[n for n, _ in _cases()])
def test_mma_kernel_tables_match_float64_fft(name, x):
    """mfcc_mma.cuh's fragment tables (mm_build_tables), exact sample split, twiddles and bin assembly."""
    x = np.asarray(x).astype(np.int16)
    ref = np.abs(np.fft.rfft(x.astype(np.float64))) ** 2
    got = _mma_power(x)
    peak = max(ref.max(), 1.0)
    assert np.max(np.abs(got - ref)) / peak < 3e-6, name
    if np.all(x == x[0]):                                              # constant frame: exact zeros outside bin 0
        assert np.all(got[1:] == 0.0)


def _mfcc_frame(pr, x512):
    from mycroft_precise_b200.core import make_config
    lib = get_lib()
    cfg = make_config(pr)
    x = np.ascontiguousarray(x512, dtype=np.int16)
    out = np.zeros(min(pr.n_filt, pr.n_mfcc), np.float32)
    rc = lib.pb_debug_tc_mfcc_frame(C.byref(cfg), x.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
    assert rc == 0, lib.pb_last_error()
    return out


@pytest.mark.parametrize('kw', [dict(), dict(n_filt=16, n_mfcc=10), dict(sample_rate=8000), dict(n_filt=22, n_mfcc=16)])
def test_full_frame_model_matches_oracle_mfcc(kw):
    """Accumulators + the kernel's epilogue (table-driven mel sums, log, DCT, c0) against the float64 oracle MFCC row."""
    from mycroft_precise_b200 import ListenerParams
    from oracle import mfcc as om
    pr = ListenerParams(**kw)
    rs = np.random.RandomState(11)
    sigs = [np.clip(rs.randn(1600) * 3000, -32768, 32767), np.zeros(1600), np.full(1600, 32767.0),
            20000 * np.sin(2 * np.pi * 700 / pr.sample_rate * np.arange(1600)), np.round(rs.randn(1600) * 3)]
    for sig in sigs:
        x = sig.astype(np.int16)
        want = om.mfcc_spec(x.astype(np.float32) / 32768.0, pr.sample_rate, 1600, 800, 512, pr.n_filt, pr.n_mfcc)[0]
        got = _mfcc_frame(pr, x[:512])
        assert got.shape == want.shape
        assert np.max(np.abs(got - want)) < 2e-4, (kw, np.max(np.abs(got - want)))


# ---------------------------------------------------------------------------------------------------------------------
# k1 mode 5 (csrc/mfcc_tc3.cuh): both DFT stages as matrix products on exactly split int16 samples
def _tc3(pr, x512, power=False):
    from mycroft_precise_b200.core import make_config
    lib = get_lib()
    cfg = make_config(pr)
    x = np.ascontiguousarray(x512, dtype=np.int16)
    out = np.zeros(min(pr.n_filt, pr.n_mfcc), np.float32)
    pw = np.zeros(257, np.float64)
    rc = lib.pb_debug_tc3_mfcc_frame(C.byref(cfg), x.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p),
                                     pw.ctypes.data_as(C.c_void_p) if power else None)
    assert rc == 0, lib.pb_last_error()
    return (out, pw) if power else out


@pytest.mark.parametrize('name,x', list(_cases()), ids=[n for n, _ in _cases()])
def test_two_stage_model_matches_float64_fft(name, x):
    from mycroft_precise_b200 import ListenerParams
    x = np.asarray(x).astype(np.int16)
    ref = np.abs(np.fft.rfft(x.astype(np.float64))) ** 2
    _, got = _tc3(ListenerParams(), x, power=True)
    peak = max(ref.max(), 1.0)
    assert np.max(np.abs(got - ref)) / peak < 3e-6, name


def test_two_stage_model_constant_input_is_exactly_zero_off_dc():
    from mycroft_precise_b200 import ListenerParams
    for c in (0, 1, -1, 127, 128, -129, 32767, -32768):
        _, pw = _tc3(ListenerParams(), np.full(512, c, np.int16), power=True)
        assert np.all(pw[1:] == 0.0), c
        assert pw[0] == (512.0 * c) ** 2, c


def test_two_stage_model_quiet_signals_near_split_boundaries():
    """Signals of a few LSB around 0 and around the balanced split's boundaries (128 + 256 k): the hi / lo pieces cancel there."""
    from mycroft_precise_b200 import ListenerParams
    rs = np.random.RandomState(5)
    for dc in (0, 127, 128, -128, 384, 20000 + 128):
        for amp in (1, 3):
            x = (dc + np.round(rs.randn(512) * amp)).astype(np.int16)
            ref = np.abs(np.fft.rfft(x.astype(np.float64))) ** 2
            _, got = _tc3(ListenerParams(), x, power=True)
            rel = np.abs(got[1:] - ref[1:]) / max(ref[1:].max(), 1e-9)
            assert rel.max() < 2e-5, (dc, amp, rel.max())


@pytest.mark.parametrize('kw', [dict(), dict(n_filt=16, n_mfcc=10), dict(sample_rate=8000), dict(n_filt=22, n_mfcc=16)])
def test_two_stage_full_frame_model_matches_oracle_mfcc(kw):
    from mycroft_precise_b200 import ListenerParams
    from oracle import mfcc as om
    pr = ListenerParams(**kw)
    rs = np.random.RandomState(11)
    sigs = [np.clip(rs.randn(1600) * 3000, -32768, 32767), np.zeros(1600), np.full(1600, 32767.0), np.full(1600, -32768.0),
            20000 * np.sin(2 * np.pi * 700 / pr.sample_rate * np.arange(1600)), np.round(rs.randn(1600) * 3),
            127 + np.round(rs.randn(1600) * 2)]
    for sig in sigs:
        x = sig.astype(np.int16)
        want = om.mfcc_spec(x.astype(np.float32) / 32768.0, pr.sample_rate, 1600, 800, 512, pr.n_filt, pr.n_mfcc)[0]
        got = _tc3(pr, x[:512])
        assert got.shape == want.shape
        assert np.max(np.abs(got - want)) < 2e-4, (kw, np.max(np.abs(got - want)))
