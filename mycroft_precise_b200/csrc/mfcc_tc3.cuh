// mfcc_tc3.cuh -- CPU model of an MFCC frame with BOTH DFT stages as fp16 matrix products (the reference's default geometry:
// n_fft 512, 20 mel filters at 16 kHz; precise/params.py:140-144).  It specifies the decomposition and splits that the tensor-core
// MFCC tick (mfcc_mma.cuh) computes; that kernel's own fragment tables and bin assembly are checked by mm_host_power.
//
// Replaces, per frame, np.fft.rfft(frame, n=512) -> power -> mel filterbank -> log -> DCT -> c0 of sonopy.mfcc_spec as the
// reference calls it (precise/vectorization.py:36-39).
//
// n = n2 + 32 q (n2 < 32, q < 16), k = 16 m + r:
//   stage 1 (matrix product): Y_r[n2] = sum_q x[n2 + 32 q] w16^(q r), r = 0..8.  The int16 samples are split EXACTLY into two fp16
//            pieces (x - x0 = 256 hi + lo, |lo| <= 128, balanced so that a quiet signal has hi = 0).
//   between:                  Z_r[n2] = Y_r[n2] w512^(n2 r), fp16 hi / lo split.
//   stage 2 (matrix product): X[16 m + r] = sum_n2 Z_r[n2] w32^(n2 m), X[16 m + 16 - r] from conj(Z_r): nine 64-column blocks
//            sharing one 64 x 64 matrix (mfcc_tc.cuh).
//   epilogue:                 power, mel edge sums, log, DCT.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "mfcc_tc.cuh"

namespace pb {

constexpr float TC3_Z_SCALE = 0.03125f;         // stage-2 operands hold Z * 2^-5 (= TCD_A_SCALE): |.| <= 32768 < fp16 max

// block r -> tile row h (of the frame's four) and MMA slot: rows hold 64, 64, 64 and 65 bins
__host__ __device__ constexpr int tc3_blk_h(int b) { constexpr int t[9] = {3, 0, 0, 1, 1, 2, 2, 3, 3}; return t[b]; }
__host__ __device__ constexpr int tc3_blk_s(int b) { constexpr int t[9] = {1, 0, 1, 0, 1, 0, 1, 0, 2}; return t[b]; }
__host__ __device__ constexpr int tc3_hs_blk(int h, int s) { constexpr int t[12] = {1, 2, -1, 3, 4, -1, 5, 6, -1, 7, 0, 8}; return t[3 * h + s]; }
// stage-2 K index of input n2 = 4 g + j inside its K-group: (re, im) adjacent -> one 4-byte store per input
__host__ __device__ constexpr int tc3_kslot(int j, int im) { return 2 * j + im; }
// stage-1 output column: 0 = Y_0, 1 = Y_8, 2 r / 2 r + 1 = Re / Im Y_r (r = 1..7)
__host__ __device__ constexpr int tc3_y_col(int r, int im) { return r == 0 ? 0 : r == 8 ? 1 : 2 * r + im; }

// ---------------------------------------------------------------------------------------------------------------------
// Host tables.
//   B1 (stage 1), four variants of [kchunk 2][n 16][8] fp16 (K-major canonical): element (column n, k = q) at
//   (q / 8) * 128 + n * 8 + q % 8.  Variants: 0 / 1 = hi / lo piece of 2^15 w (multiplies the hi piece of x, stored / 128),
//   2 / 3 = hi / lo piece of w (multiplies the lo piece of x).
static inline void tc3_build_b1(std::vector<__half>& b1) {
    b1.assign((size_t)4 * 256, __float2half_rn(0.f));
    const double PI2 = 6.283185307179586476925286766559;
    for (int q = 0; q < 16; ++q)
        for (int n = 0; n < 16; ++n) {
            double v;
            if (n == 0) v = 1.0;
            else if (n == 1) v = (q & 1) ? -1.0 : 1.0;
            else {
                const int r = n >> 1;
                const double a = PI2 * ((q * r) & 15) / 16.0;
                v = (n & 1) ? -sin(a) : cos(a);
            }
            for (int var = 0; var < 2; ++var) {
                const double sv = var == 0 ? v * 32768.0 : v;
                const __half hi = __float2half_rn((float)sv);
                const __half lo = __float2half_rn((float)(sv - (double)__half2float(hi)));
                const size_t o = (size_t)(q >> 3) * 128 + (size_t)n * 8 + (q & 7);
                b1[(size_t)(2 * var) * 256 + o] = hi;
                b1[(size_t)(2 * var + 1) * 256 + o] = lo;
            }
        }
}
//   B2 (stage 2): the 64 x 64 matrix of mfcc_tc.cuh with the K order of this model (tc3_kslot), pieces hi then lo.
static inline void tc3_build_b2(std::vector<__half>& b2) {
    b2.assign((size_t)2 * 8 * 64 * 8, __float2half_rn(0.f));
    const double PI2 = 6.283185307179586476925286766559;
    for (int g = 0; g < 8; ++g)
        for (int j = 0; j < 4; ++j)
            for (int im = 0; im < 2; ++im)
                for (int n = 0; n < 64; ++n) {
                    const int n2 = 4 * g + j, quarter = n >> 4, m = n & 15;
                    const double a = PI2 * n2 * (quarter < 2 ? m : m + 1) / 32.0;
                    const double tr = cos(a), ti = -sin(a);
                    double v;
                    if (quarter == 0) v = im ? -ti : tr;
                    else if (quarter == 1) v = im ? tr : ti;
                    else if (quarter == 2) v = im ? ti : tr;
                    else v = im ? -tr : ti;
                    const __half hi = __float2half_rn((float)v);
                    const __half lo = __float2half_rn((float)(v - (double)__half2float(hi)));
                    const size_t o = ((size_t)g * 64 + n) * 8 + tc3_kslot(j, im);
                    b2[o] = hi; b2[(size_t)8 * 64 * 8 + o] = lo;
                }
}
//   Twiddles of input n2: tw[n2 * 16 + 2 (r - 1)] = 2^-5 (cos, -sin)(2 pi n2 r / 512), r = 1..8.
static inline void tc3_build_tw(std::vector<float>& tw) {
    tw.assign((size_t)32 * 16, 0.f);
    const double PI2 = 6.283185307179586476925286766559;
    for (int n2 = 0; n2 < 32; ++n2)
        for (int r = 1; r <= 8; ++r) {
            const double a = PI2 * n2 * r / 512.0;
            tw[(size_t)n2 * 16 + 2 * (r - 1)] = (float)(cos(a) * (double)TC3_Z_SCALE);
            tw[(size_t)n2 * 16 + 2 * (r - 1) + 1] = (float)(-sin(a) * (double)TC3_Z_SCALE);
        }
}

// balanced split of an int16: x = 256 hi + lo, lo in [-128, 127]
__host__ __device__ __forceinline__ void tc3_split16(int x, int& hi, int& lo) {
    lo = (((x & 255) ^ 128) - 128);
    hi = (x - lo) >> 8;
}

// The twiddle + scale step for one input: y[16] (tc3_y_col order) -> zr / zi of blocks 0..8.  Host + device.
__host__ __device__ __forceinline__ void tc3_twiddle(const float (&y)[16], const float (&tw)[16], float (&zr)[9], float (&zi)[9]) {
    zr[0] = y[0] * TC3_Z_SCALE; zi[0] = 0.f;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int r = 1; r < 8; ++r) {
        const float c = tw[2 * (r - 1)], s = tw[2 * (r - 1) + 1];
        zr[r] = fmaf(y[2 * r], c, -(y[2 * r + 1] * s));
        zi[r] = fmaf(y[2 * r], s, y[2 * r + 1] * c);
    }
    zr[8] = y[1] * tw[14]; zi[8] = y[1] * tw[15];
}

// CPU model of the arithmetic for ONE frame of 512 int16 samples (same splits, tables, pass order and layout
// arithmetic; fp16 products accumulated in fp32): d[9][64] = the frame's stage-2 accumulator columns block by block, X[0]
// restored.  What tests/test_tc_dft_host_model.py checks without a device.
static inline void tc3_host_accumulators(const int16_t* x, float (*d)[64]) {
    static std::vector<__half> b1, b2;
    static std::vector<float> tw;
    if (b1.empty()) { tc3_build_b1(b1); tc3_build_b2(b2); tc3_build_tw(tw); }
    int hi0, lo0;
    tc3_split16(x[0], hi0, lo0);
    std::vector<float> a((size_t)TCD_BLOCKS * 64);
    for (int n2 = 0; n2 < 32; ++n2) {
        float y[16];
        for (int n = 0; n < 16; ++n) {
            float acc = 0.f;
            for (int pass = 0; pass < 4; ++pass) {            // lo x w_lo, lo x w_hi, hi x W_lo, hi x W_hi
                float part = 0.f;
                for (int q = 0; q < 16; ++q) {
                    int hi, lo;
                    tc3_split16(x[n2 + 32 * q], hi, lo);
                    const float av = pass < 2 ? (float)(lo - lo0) : (float)(hi - hi0) * 0.0078125f;
                    const int var = pass == 0 ? 3 : pass == 1 ? 2 : pass == 2 ? 1 : 0;
                    const size_t o = (size_t)var * 256 + (size_t)(q >> 3) * 128 + (size_t)n * 8 + (q & 7);
                    part += av * __half2float(b1[o]);
                }
                acc += part;
            }
            y[n] = acc;
        }
        float twl[16], zr[9], zi[9];
        for (int e = 0; e < 16; ++e) twl[e] = tw[(size_t)n2 * 16 + e];
        tc3_twiddle(y, twl, zr, zi);
        const int g = n2 >> 2, j = n2 & 3;
        for (int b = 0; b < TCD_BLOCKS; ++b) { a[b * 64 + 8 * g + tc3_kslot(j, 0)] = zr[b]; a[b * 64 + 8 * g + tc3_kslot(j, 1)] = zi[b]; }
    }
    for (int b = 0; b < TCD_BLOCKS; ++b)
        for (int n = 0; n < 64; ++n) {
            float acc = 0.f;
            for (int pass = 0; pass < 3; ++pass)
                for (int k = 0; k < 64; ++k) {
                    const float av = a[b * 64 + k];
                    const __half ah = __float2half_rn(av);
                    const __half al = __float2half_rn(av - __half2float(ah));
                    const size_t o = ((size_t)(k >> 3) * 64 + n) * 8 + (k & 7);
                    const float pa = __half2float(pass == 0 ? al : ah);
                    const float pb = __half2float(pass == 1 ? b2[(size_t)8 * 64 * 8 + o] : b2[o]);
                    acc += pa * pb;
                }
            d[b][n] = acc;
        }
    d[0][0] += TCD_X0_D * (float)x[0];
}

// The epilogue's arithmetic for one frame (fp32), in this order: per segment s = 1..19 the power sum and the
// rising-edge sum (falling edge = sum - rising), segment 20 with its falling weights, log, DCT, c0.
static inline void tc3_host_epilogue(const float (*d)[64], const std::vector<float>& wrise, const std::vector<float>& wfall,
                                     const std::vector<int>& grid, const float* dct, int n_filt, int n_out, float pscale, float* out) {
    float rise[TCD_MAX_FILT + 2] = {0}, seg[TCD_MAX_FILT + 2] = {0}, fall_last = 0.f;
    for (int b = 0; b < TCD_BLOCKS; ++b)
        for (int half = 0; half < 2; ++half)
            for (int m = 0; m < 16; ++m) {
                const int k = tcd_col_bin(b, 32 * half + m);
                if (k < 0) continue;
                const float re = d[b][32 * half + m], im = d[b][32 * half + 16 + m];
                const float p = (k == 0 || k == 256) ? re * re : fmaf(im, im, re * re);
                int s = 0;
                while (s < n_filt && k >= grid[s + 1]) ++s;
                seg[s] += p;
                if (s < n_filt) rise[s] = fmaf(wrise[k], p, rise[s]);
                else fall_last = fmaf(wfall[k], p, fall_last);
            }
    const float eps = 2.220446049250313e-16f;
    float lg[TCD_MAX_FILT], tot = 0.f;
    for (int s = 0; s <= n_filt; ++s) tot += seg[s];
    for (int j = 0; j < n_filt; ++j) {
        const float fall = j + 1 < n_filt ? seg[j + 1] - rise[j + 1] : fall_last;
        lg[j] = logf(fmaxf((rise[j] + fall) * pscale, eps));
    }
    for (int o = 0; o < n_out; ++o) {
        float v = 0.f;
        for (int j = 0; j < n_filt; ++j) v = fmaf(dct[(size_t)o * 24 + j], lg[j], v);
        out[o] = o == 0 ? logf(fmaxf(tot * pscale, eps)) : v;
    }
}

}  // namespace pb
