"""CPU: the numerical design study for the round-2 tensor-core DFT (scripts/proto_tc_dft.py) stays valid: the block twiddle
matrices, the accumulator-column -> bin map and the fp16 hi/lo three-pass scheme reproduce a float64 power spectrum."""
import importlib.util
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _proto():
    spec = importlib.util.spec_from_file_location('proto_tc_dft', os.path.join(ROOT, 'scripts', 'proto_tc_dft.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_radix16_block_formulation_matches_float64_fft():
    p = _proto()
    assert p.check_radix16() < 5e-6
    cols = p.column_bins()
    used = sorted(c for pair in cols for c in pair if c >= 0)
    assert len(cols) == 257 and used == list(range(512))          # every accumulator column is exactly one bin component


def test_radix4_three_pass_matches_float64_fft():
    p = _proto()
    rs = np.random.RandomState(3)
    x = np.clip(rs.randn(8, 512) * 3000, -32768, 32767).astype(np.int16)
    ref = np.abs(np.fft.rfft(x.astype(np.float64), axis=1)) ** 2
    for passes, tol in ((3, 5e-6), (1, 1e-2)):
        got = p.tc_power(x, passes)
        err = np.max(np.abs(got - ref) / ref.max(axis=1, keepdims=True))
        assert err < tol
    assert np.max(np.abs(p.tc_power(x, 1) - ref) / ref.max(axis=1, keepdims=True)) > 1e-5      # one fp16 pass is not enough


def _frames_ready(n, used, hop):
    return (n - used) // hop + 1 if n >= used else 0


def test_tensor_core_tick_state_machine_claims():
    """The experimental kernel (csrc/mfcc_tc.cuh) simplifies the stream state machine of the fast kernel under
    chunk >= 512, chunk % 8 == 0, hop % 8 == 0: nothing of the old tail survives a tick, every frame is the concatenation of
    at most one tail piece and one chunk piece whose lengths and offsets are multiples of 4 samples (8-byte vector loads), and
    the new tail is a multiple of 8 samples (16-byte vector copies).  Transcribes the kernel's index arithmetic and checks it
    against the ground truth on a sample-indexed signal."""
    used = 512
    for hop, chunk in ((800, 1024), (800, 512), (800, 2048), (400, 1024), (160, 512), (808, 1000), (800, 1600), (1024, 1024)):
        assert chunk % 8 == 0 and hop % 8 == 0 and chunk >= 512
        sig = np.arange(40 * chunk, dtype=np.int64)              # sample value == absolute index
        n0, tail, ts_tail = 0, np.zeros(0, np.int64), 0
        produced = 0
        for k in range(40):
            ch = sig[k * chunk:(k + 1) * chunk]
            c0 = _frames_ready(n0, used, hop)
            cnt = _frames_ready(n0 + chunk, used, hop) - c0
            assert cnt <= (chunk + hop - 1) // hop
            ts0 = min(c0 * hop, n0)
            assert ts0 == ts_tail and len(tail) == n0 - ts0 and len(tail) < 512
            assert -512 < c0 * hop - n0 <= max(hop - 512, 0) or n0 < used      # the LEAN fast kernel packs this into 32 bits
            for sub in range(cnt):
                a0 = (c0 + sub) * hop
                if a0 >= n0:
                    len0, p0, p1 = 0, None, a0 - n0
                else:
                    len0, p0, p1 = min(used, n0 - a0), a0 - ts0, 0
                    assert p0 % 4 == 0
                    assert ts0 == c0 * hop and p0 == sub * hop        # LEAN: offset inside the tail = sub * hop
                assert len0 % 4 == 0 and p1 % 4 == 0
                got = np.empty(512, np.int64)
                for g in range(8):                                # the producer's loads: 4 samples at i = 4 g + 32 q
                    for q in range(16):
                        i = 4 * g + 32 * q
                        src = tail[p0 + i:p0 + i + 4] if i < len0 else ch[p1 + i - len0:p1 + i - len0 + 4]
                        got[i:i + 4] = src
                assert np.array_equal(got, sig[a0:a0 + 512]), (hop, chunk, k, sub)
                produced += 1
            n1 = n0 + chunk
            c1 = c0 + cnt
            ts1 = min(c1 * hop, n1)
            assert ts1 >= n0, 'part of the old tail would have to survive'
            assert (n1 - ts1) % 8 == 0 and n1 - ts1 < 512 and (ts1 - n0) % 8 == 0
            tail, ts_tail, n0 = ch[ts1 - n0:], ts1, n1
        assert produced == _frames_ready(n0, used, hop)

