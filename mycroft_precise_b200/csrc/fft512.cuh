// fft512.cuh -- register-resident 512-point real FFT -> power spectrum, 16 lanes per frame.
//
// Replaces, per frame, np.fft.rfft(frame, n=512) and (re^2+im^2)/512 inside sonopy.power_spec
// as the reference calls it (precise/vectorization.py:36-39).
//
// Decomposition.  The 512 real samples are packed as 256 complex z[m] = x[2m] + i x[2m+1];
// Z = FFT256(z) is computed as 16 x 16 (m = 16 n1 + n2, k = k1 + 16 k2):
//
//   stage 1 (lane = n2): Y[k1] = sum_n1 W16^(n1 k1) z[16 n1 + n2]      in-lane FFT-16
//   twiddle            : Y[k1] *= W256^(n2 k1)                          per-lane constants
//   exchange           : 16x16 transpose of the half-warp through padded shared memory
//   stage 2 (lane = k1): Z[k1+16k2] = sum_n2 W16^(n2 k2) Y'[n2]         in-lane FFT-16
//
// The real-input split needs Z[k] and Z[256-k] together; bin k = k1 + 16 k2 lives in lane k1,
// its mirror in lane (16-k1)%16, element 15-k2 ((16-k2)%16 for lane 0).  Each lane handles the
// pairs of its own elements k2 = 0..7 (the mirror lane handles the other eight), fetching the
// partner with two shuffles, and emits both bins of the pair from
//     |X[k]|^2, |X[256-k]|^2 = (|E|^2 + |O|^2) +- 2 Re(E conj(w O)),   w = W512^k.
#pragma once
#include <cuda_runtime.h>

namespace pb {

struct cpx { float x, y; };

__device__ __forceinline__ cpx cadd(cpx a, cpx b) { return {a.x + b.x, a.y + b.y}; }
__device__ __forceinline__ cpx csub(cpx a, cpx b) { return {a.x - b.x, a.y - b.y}; }
// a * (wr + i wi)
__device__ __forceinline__ cpx cmul(cpx a, float wr, float wi) {
    return {fmaf(a.x, wr, -a.y * wi), fmaf(a.x, wi, a.y * wr)};
}
// a * (-i)
__device__ __forceinline__ cpx cmul_mi(cpx a) { return {a.y, -a.x}; }

// forward 4-point DFT, in place, natural order
__device__ __forceinline__ void fft4(cpx& a0, cpx& a1, cpx& a2, cpx& a3) {
    cpx s0 = cadd(a0, a2), s1 = csub(a0, a2), s2 = cadd(a1, a3), s3 = cmul_mi(csub(a1, a3));
    a0 = cadd(s0, s2); a2 = csub(s0, s2); a1 = cadd(s1, s3); a3 = csub(s1, s3);
}

#define PB_C1 0.92387953251128674f   // cos(pi/8)
#define PB_S1 0.38268343236508977f   // sin(pi/8)
#define PB_R2 0.70710678118654752f   // sqrt(1/2)

// forward 16-point DFT of a[0..15] (a[n]), result X[k] returned in a[k].  Radix 4 x 4:
// n = 4 na + nb, k = ka + 4 kb.
__device__ __forceinline__ void fft16(cpx (&a)[16]) {
    // first pass: for each nb, FFT-4 over na of a[4 na + nb] -> t[nb][ka] stored at a[4 ka + nb]
#pragma unroll
    for (int nb = 0; nb < 4; ++nb) fft4(a[nb], a[4 + nb], a[8 + nb], a[12 + nb]);
    // twiddles W16^(nb ka) on a[4 ka + nb]
    a[4 + 1] = cmul(a[4 + 1], PB_C1, -PB_S1);                 // W^1
    a[4 + 2] = cmul(a[4 + 2], PB_R2, -PB_R2);                 // W^2
    a[4 + 3] = cmul(a[4 + 3], PB_S1, -PB_C1);                 // W^3
    a[8 + 1] = cmul(a[8 + 1], PB_R2, -PB_R2);                 // W^2
    a[8 + 2] = cmul_mi(a[8 + 2]);                             // W^4 = -i
    a[8 + 3] = cmul(a[8 + 3], -PB_R2, -PB_R2);                // W^6
    a[12 + 1] = cmul(a[12 + 1], PB_S1, -PB_C1);               // W^3
    a[12 + 2] = cmul(a[12 + 2], -PB_R2, -PB_R2);              // W^6
    a[12 + 3] = cmul(a[12 + 3], -PB_C1, PB_S1);               // W^9
    // second pass: for each ka, FFT-4 over nb of a[4 ka + nb] -> X[ka + 4 kb] left at a[4 ka + kb]
#pragma unroll
    for (int ka = 0; ka < 4; ++ka) fft4(a[4 * ka], a[4 * ka + 1], a[4 * ka + 2], a[4 * ka + 3]);
    // a[4 ka + kb] holds X[ka + 4 kb]: transpose the 4x4 index grid into natural order
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = i + 1; j < 4; ++j) { cpx t = a[4 * i + j]; a[4 * i + j] = a[4 * j + i]; a[4 * j + i] = t; }
}

constexpr int XCH_STRIDE = 17;                 // complex elements per padded row
constexpr int XCH_ELEMS = 16 * XCH_STRIDE;     // per frame
constexpr int NBINS512 = 257;

// Per-lane constants, loaded once per thread.
struct FftLaneConst {
    float twr[16], twi[16];   // W256^(n2 k1), k1 = 0..15 (lane = n2)
    float pcr, psi;           // cos/sin(2 pi k1 / 512)            (lane = k1)
    static constexpr bool kSplitXch = false;
    __device__ __forceinline__ float2 tw(int k) const { return make_float2(twr[k], twi[k]); }
};

// The same constants with the stage twiddles read from shared memory instead of 32 registers: tws = a [k1][16] float2
// table (W256^(n2 k1) at tws[16 k1 + n2]) plus this lane's n2, so the 16 lanes of a half-warp read 16 consecutive float2.
// Its exchange goes through a float [16][XCH_STRIDE] scratch, one component at a time (half the shared memory).
struct FftSmemConst {
    const float2* tws;
    float pcr, psi;
    static constexpr bool kSplitXch = true;
    __device__ __forceinline__ float2 tw(int k) const { return tws[16 * k]; }
};

__device__ __forceinline__ void load_lane_const(FftLaneConst& c, const float2* __restrict__ tw_stage,
                                                const float2* __restrict__ tw_post, int l16) {
#pragma unroll
    for (int k = 0; k < 16; ++k) { float2 t = tw_stage[l16 * 16 + k]; c.twr[k] = t.x; c.twi[k] = t.y; }
    float2 p = tw_post[l16];
    c.pcr = p.x; c.psi = p.y;
}

// cos/sin(2 pi k2 / 32), k2 = 0..8
__device__ __forceinline__ void w32(int k2, float& c, float& s) {
    constexpr float C[9] = {1.f, 0.98078528040323043f, 0.92387953251128674f, 0.83146961230254524f,
                            0.70710678118654752f, 0.55557023301960218f, 0.38268343236508977f,
                            0.19509032201612825f, 0.f};
    constexpr float S[9] = {0.f, 0.19509032201612825f, 0.38268343236508977f, 0.55557023301960218f,
                            0.70710678118654752f, 0.83146961230254524f, 0.92387953251128674f,
                            0.98078528040323043f, 1.f};
    c = C[k2]; s = S[k2];
}

// One frame per half-warp.  z[n1] = packed complex element 16 n1 + l16 of this lane's frame
// (inactive half-warps pass zeros and `active` = false; all 32 lanes must call).
// xch: this half-warp's scratch, XCH_ELEMS float2 (FftLaneConst) or XCH_ELEMS floats (FftSmemConst).  P: this frame's power
// row (>= 257 floats).  scale multiplies |X|^2 (1/512 and the int16 -> float normalisation folded together).
template <class Const>
__device__ __forceinline__ void fft512_power(cpx (&z)[16], const Const& c, void* xch,
                                             float* P, float scale, int l16, bool active) {
    const unsigned FULL = 0xffffffffu;
    fft16(z);
#pragma unroll
    for (int k = 1; k < 16; ++k) { const float2 w = c.tw(k); z[k] = cmul(z[k], w.x, w.y); }
    if (Const::kSplitXch) {
        float* x = static_cast<float*>(xch);
#pragma unroll
        for (int k = 0; k < 16; ++k) x[k * XCH_STRIDE + l16] = z[k].x;
        __syncwarp();
#pragma unroll
        for (int n = 0; n < 16; ++n) z[n].x = x[l16 * XCH_STRIDE + n];
        __syncwarp();
#pragma unroll
        for (int k = 0; k < 16; ++k) x[k * XCH_STRIDE + l16] = z[k].y;
        __syncwarp();
#pragma unroll
        for (int n = 0; n < 16; ++n) z[n].y = x[l16 * XCH_STRIDE + n];
    } else {
        float2* x = static_cast<float2*>(xch);
#pragma unroll
        for (int k = 0; k < 16; ++k) x[k * XCH_STRIDE + l16] = make_float2(z[k].x, z[k].y);
        __syncwarp();
#pragma unroll
        for (int n = 0; n < 16; ++n) { float2 t = x[l16 * XCH_STRIDE + n]; z[n].x = t.x; z[n].y = t.y; }
    }
    __syncwarp();
    fft16(z);                                  // z[k2] = Z[l16 + 16 k2]
    const int lane = threadIdx.x & 31;
    const int src = (lane & 16) | ((16 - l16) & 15);
    const float qs = 0.25f * scale;
#pragma unroll
    for (int k2 = 0; k2 < 8; ++k2) {
        // value this lane sends: its element mirrored for the receiver's k2
        cpx snd = (l16 == 0) ? z[(16 - k2) & 15] : z[15 - k2];
        cpx b;
        b.x = __shfl_sync(FULL, snd.x, src);
        b.y = __shfl_sync(FULL, snd.y, src);
        cpx a = z[k2];
        float er = a.x + b.x, ei = a.y - b.y;          // 2E = a + conj(b)
        float orr = a.y + b.y, oi = b.x - a.x;         // 2O = (a - conj(b)) / i
        float ck, sk; w32(k2, ck, sk);
        float cw = fmaf(c.pcr, ck, -c.psi * sk);       // cos(2 pi k / 512), k = l16 + 16 k2
        float sw = fmaf(c.psi, ck, c.pcr * sk);        // sin
        float tr = fmaf(cw, orr, sw * oi);             // 2 w O, w = cw - i sw
        float ti = fmaf(cw, oi, -sw * orr);
        float A = fmaf(er, er, fmaf(ei, ei, fmaf(orr, orr, oi * oi)));
        float B = 2.f * fmaf(er, tr, ei * ti);
        if (active) {
            int k = l16 + 16 * k2;
            P[k] = (A + B) * qs;
            P[256 - k] = (A - B) * qs;
        }
    }
    if (active && l16 == 0) P[128] = fmaf(z[8].x, z[8].x, z[8].y * z[8].y) * scale;
}

}  // namespace pb
