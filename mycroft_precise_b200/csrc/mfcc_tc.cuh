// mfcc_tc.cuh -- host tables and CPU model of an MFCC frame whose second DFT stage is an fp16 matrix product (the shape a
// tensor-core MFCC tick computes: mfcc_mma.cuh, k1 mode 4).
//
// Replaces, per frame, np.fft.rfft(frame, n=512), the power spectrum, the mel filterbank, log, DCT and c0 of
// sonopy.mfcc_spec as the reference calls it (precise/vectorization.py:36-39), for the stateful tick
// (Listener.update_vectors, precise/network_runner.py:125-146).
//
// Decomposition.  n = n2 + 32 q (n2 < 32, q < 16), k = 16 m + r:
//     Y_r[n2]     = sum_q x[n2 + 32 q] w16^(q r)          r = 0..8     16-point DFT of REAL data        CUDA cores (fp32)
//     Z_r[n2]     = Y_r[n2] w512^(n2 r)                                twiddle                          CUDA cores (fp32)
//     X[16 m + r]      = sum_n2       Z_r[n2]  w32^(n2 m)                                               tensor cores
//     X[16 m + 16 - r] = sum_n2 conj(Z_r[n2]) w32^(n2 (m + 1))         (conj(Y_r) = Y_(16-r))           tensor cores
// Because the twiddle is applied before the GEMM, every block r = 0..8 multiplies the SAME 64 x 64 real matrix (rows: Re Z,
// Im Z of the 32 inputs; columns: Re, Im of X[16 m + r], then Re, Im of X[16 m + 16 - r]); 16 KB of operands instead of one
// 64 x 64 matrix per block (128 KB), which is what leaves shared memory for staging the PCM by bulk copies and lets four
// blocks of a frame be stacked along M (a tile is 32 frames x 4 rows).  Block 0 (Z_0 = Y_0, real) yields X[16 m] and, in the
// second half at m = 15, X[256]; block 8 yields X[16 m + 8].  Operands are fp16 hi + lo pieces, three passes
// (a_lo b_hi + a_hi b_lo + a_hi b_hi, fp32 accumulate): ~1e-6 of the peak bin against a float64 FFT.
// The CPU model below (same butterfly, same twiddles, same operand tables read through the same layout arithmetic) is
// what tests/test_tc_dft_host_model.py checks without a device.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <vector>


namespace pb {

constexpr int TCD_BLOCKS = 9;                 // GEMM blocks per frame, r = 0..8
constexpr int TCD_KSTEPS = 4;                 // K = 64 per block = 4 MMA K-steps of 16
constexpr int TCD_MAX_FILT = 22;
constexpr int TCD_MAX_OUT = 16;
constexpr int TCD_TW_STRIDE = 18;             // floats per input n2 in the twiddle table: (cos, -sin) of r = 1..8, + 2 of padding
constexpr float TCD_IN_SCALE = 0.015625f;     // 2^-6 folded into the int16 -> float conversion; the butterfly returns 2 Y
constexpr float TCD_A_SCALE = 0.03125f;       // => A operands hold Z * 2^-5: |A| <= 16384, and <= 32768 < fp16 max after the shift below
// The model transforms x - x[0] (a constant only moves X[0]; constant input then gives exact zeros everywhere else, like the
// float64 reference and the FFT kernels): Y_0 loses 16 x[0], i.e. the butterfly output 2 * 16 * IN_SCALE * x[0], and the
// X[0] accumulator gets 32 times that back.
constexpr float TCD_X0_Y = 32.f * TCD_IN_SCALE;          // 0.5
constexpr float TCD_X0_D = 32.f * TCD_X0_Y;              // 16

// A tile row is (frame, h), h = 0..3; row h carries up to three blocks in the MMA "slots" 0..2 (64 accumulator columns each).
__host__ __device__ constexpr int tcd_blk_h(int b) { constexpr int t[9] = {0, 0, 0, 1, 1, 2, 2, 3, 1}; return t[b]; }
__host__ __device__ constexpr int tcd_blk_s(int b) { constexpr int t[9] = {2, 0, 1, 0, 1, 0, 1, 0, 2}; return t[b]; }
__host__ __device__ constexpr int tcd_hs_blk(int h, int s) { constexpr int t[12] = {1, 2, 0, 3, 4, 8, 5, 6, -1, 7, -1, -1}; return t[3 * h + s]; }
// position (0..7) inside K-group g (inputs n2 = 4 g .. 4 g + 3) of input n2 = 4 g + j, real (im = 0) or imaginary part:
// two 8-byte halves, one per sample pair (j >> 1), swapped for odd g so that the lanes of a half-warp (4 K-groups x 4
// frames) store to 16 different 8-byte bank groups
__host__ __device__ constexpr int tcd_kslot(int j, int im, int g) { return 4 * ((j >> 1) ^ (g & 1)) + 2 * im + (j & 1); }
// bin held by column c of block b (quarter c >> 4: Re / Im of X[16 m + b], Re / Im of X[16 m + 16 - b]; m = c & 15), or -1
// where the column repeats another block's bin (second halves of blocks 0 and 8, except X[256] in block 0)
__host__ __device__ constexpr int tcd_col_bin(int b, int c) {
    const int m = c & 15, second = c >> 5;
    if (b == 0) return second ? (m == 15 ? 256 : -1) : 16 * m;
    if (b == 8) return second ? -1 : 16 * m + 8;
    return second ? 16 * m + 16 - b : 16 * m + b;
}

// ---------------------------------------------------------------------------------------------------------------------
// 16-point DFT of real data, outputs scaled by 2: yr[k] + i yi[k] = 2 * sum_q x[q] w16^(q k), k = 0..8 (yi[0] = yi[8] = 0).
// Packed as an 8-point complex FFT of z[n] = x[2n] + i x[2n+1] plus the real-input split.  Host + device: the CPU tests call
// the host build of exactly this function.
__host__ __device__ __forceinline__ void rdft16_x2(const float (&x)[16], float (&yr)[9], float (&yi)[9]) {
    const float R = 0.70710678118654752f, C1 = 0.92387953251128674f, S1 = 0.38268343236508977f;
    // FFT8 of z: even part (z0 z2 z4 z6), odd part (z1 z3 z5 z7)
    float er[4], ei[4], orr[4], oi[4];
    {
        const float ar = x[0] + x[8], ai = x[1] + x[9], br = x[0] - x[8], bi = x[1] - x[9];          // z0 +- z4
        const float cr = x[4] + x[12], ci = x[5] + x[13], dr = x[4] - x[12], di = x[5] - x[13];      // z2 +- z6
        er[0] = ar + cr; ei[0] = ai + ci; er[2] = ar - cr; ei[2] = ai - ci;
        er[1] = br + di; ei[1] = bi - dr; er[3] = br - di; ei[3] = bi + dr;                          // -i (z2 - z6) = (di, -dr)
    }
    {
        const float ar = x[2] + x[10], ai = x[3] + x[11], br = x[2] - x[10], bi = x[3] - x[11];      // z1 +- z5
        const float cr = x[6] + x[14], ci = x[7] + x[15], dr = x[6] - x[14], di = x[7] - x[15];      // z3 +- z7
        orr[0] = ar + cr; oi[0] = ai + ci; orr[2] = ar - cr; oi[2] = ai - ci;
        orr[1] = br + di; oi[1] = bi - dr; orr[3] = br - di; oi[3] = bi + dr;
    }
    // Z[k] = E[k] + w8^k O[k], Z[k+4] = E[k] - w8^k O[k];  w8 = (1 - i) / sqrt 2, w8^2 = -i, w8^3 = (-1 - i) / sqrt 2
    float zr[8], zi[8];
    {
        float tr = orr[0], ti = oi[0];
        zr[0] = er[0] + tr; zi[0] = ei[0] + ti; zr[4] = er[0] - tr; zi[4] = ei[0] - ti;
        tr = (orr[1] + oi[1]) * R; ti = (oi[1] - orr[1]) * R;
        zr[1] = er[1] + tr; zi[1] = ei[1] + ti; zr[5] = er[1] - tr; zi[5] = ei[1] - ti;
        tr = oi[2]; ti = -orr[2];
        zr[2] = er[2] + tr; zi[2] = ei[2] + ti; zr[6] = er[2] - tr; zi[6] = ei[2] - ti;
        tr = (oi[3] - orr[3]) * R; ti = -(orr[3] + oi[3]) * R;
        zr[3] = er[3] + tr; zi[3] = ei[3] + ti; zr[7] = er[3] - tr; zi[7] = ei[3] - ti;
    }
    // real-input split: 2 Y[k] = S + T, S = Z[k] + conj(Z[8-k]), T = -i w16^k (Z[k] - conj(Z[8-k]))
    yr[0] = 2.f * (zr[0] + zi[0]); yi[0] = 0.f;
    yr[8] = 2.f * (zr[0] - zi[0]); yi[8] = 0.f;
    yr[4] = 2.f * zr[4]; yi[4] = -2.f * zi[4];
    const float cs[3] = {C1, R, S1}, sn[3] = {S1, R, C1};                  // cos, sin of 2 pi k / 16, k = 1, 2, 3
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int k = 1; k <= 3; ++k) {
        const float sr = zr[k] + zr[8 - k], si = zi[k] - zi[8 - k];        // S = Z[k] + conj(Z[8-k])
        const float dr = zr[k] - zr[8 - k], di = zi[k] + zi[8 - k];        // D = Z[k] - conj(Z[8-k])
        const float p1 = sn[k - 1] * dr - cs[k - 1] * di, p2 = sn[k - 1] * di + cs[k - 1] * dr;
        yr[k] = sr - p1; yi[k] = si - p2;                                  // T_k = -p1 - i p2
        yr[8 - k] = sr + p1; yi[8 - k] = -si - p2;                         // S_(8-k) = conj(S), T_(8-k) = p1 - i p2
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Host tables.
//   B operand, piece hi / lo: fp16 [kgroup 8][n 64][8]  (K-major canonical, no swizzle: element (n, k) at
//   ((k / 8) * 64 + n) * 8 + k % 8), k = 8 g + tcd_kslot(j, im, g) <-> input n2 = 4 g + j, part im.
//   Twiddles: tw[n2 * TCD_TW_STRIDE + 2 (r - 1)] = (cos, -sin)(2 pi n2 r / 512), r = 1..8.
static inline void tcd_build_b(std::vector<__half>& b_hi, std::vector<__half>& b_lo) {
    b_hi.assign((size_t)8 * 64 * 8, __float2half_rn(0.f));
    b_lo = b_hi;
    const double PI2 = 6.283185307179586476925286766559;
    for (int g = 0; g < 8; ++g)
        for (int j = 0; j < 4; ++j)
            for (int im = 0; im < 2; ++im)
                for (int n = 0; n < 64; ++n) {
                    const int n2 = 4 * g + j, quarter = n >> 4, m = n & 15;
                    const double a = PI2 * n2 * (quarter < 2 ? m : m + 1) / 32.0;
                    const double tr = cos(a), ti = -sin(a);                                 // T = w32^(n2 m) or w32^(n2 (m + 1))
                    // quarters 0, 1: (a + i b) T -> re: a tr - b ti, im: a ti + b tr
                    // quarters 2, 3: (a - i b) T -> re: a tr + b ti, im: a ti - b tr
                    double v;
                    if (quarter == 0) v = im ? -ti : tr;
                    else if (quarter == 1) v = im ? tr : ti;
                    else if (quarter == 2) v = im ? ti : tr;
                    else v = im ? -tr : ti;
                    const __half hi = __float2half_rn((float)v);
                    const __half lo = __float2half_rn((float)(v - (double)__half2float(hi)));
                    const size_t o = ((size_t)g * 64 + n) * 8 + tcd_kslot(j, im, g);
                    b_hi[o] = hi; b_lo[o] = lo;
                }
}

static inline void tcd_build_tw(std::vector<float>& tw) {
    tw.assign((size_t)32 * TCD_TW_STRIDE, 0.f);
    const double PI2 = 6.283185307179586476925286766559;
    for (int n2 = 0; n2 < 32; ++n2)
        for (int r = 1; r <= 8; ++r) {
            const double a = PI2 * n2 * r / 512.0;
            tw[(size_t)n2 * TCD_TW_STRIDE + 2 * (r - 1)] = (float)cos(a);
            tw[(size_t)n2 * TCD_TW_STRIDE + 2 * (r - 1) + 1] = (float)-sin(a);
        }
}

// One input's nine block operands from its 16-point DFT (yr, yi scaled as rdft16_x2 returns them): Z_0 = Y_0 - shift (real),
// Z_r = Y_r w512^(n2 r).  Host + device.
__host__ __device__ __forceinline__ void tcd_twiddle(const float (&yr)[9], const float (&yi)[9], const float* tw, float x0_shift,
                                                     float (&zr)[9], float (&zi)[9]) {
    zr[0] = yr[0] - x0_shift; zi[0] = 0.f;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int r = 1; r < 8; ++r) {
        const float c = tw[2 * (r - 1)], s = tw[2 * (r - 1) + 1];
        zr[r] = fmaf(yr[r], c, -(yi[r] * s));
        zi[r] = fmaf(yr[r], s, yi[r] * c);
    }
    zr[8] = yr[8] * tw[14]; zi[8] = yr[8] * tw[15];
}

// wrise / wfall / grid as built by api.cu (build_mel); pscale turns (re^2 + im^2) of the scaled accumulators into power / n_fft.
// etab[k] = (rising-edge weight, falling-edge weight, segment) of bin k  (CPU model of the epilogue)
static inline void tcd_build_etab(std::vector<float4>& etab, const std::vector<float>& wrise, const std::vector<float>& wfall,
                                  const std::vector<int>& grid, int n_filt, float pscale) {
    etab.assign(257, make_float4(0.f, 0.f, 0.f, 0.f));
    for (int k = 0; k < 257; ++k) {
        int s = 0;
        float wr = 0.f, wf = 0.f;
        if (k >= grid[0] && k < grid[n_filt + 1]) {
            while (s < n_filt && k >= grid[s + 1]) ++s;                 // segment: grid[s] <= k < grid[s + 1]
            if (s < n_filt) wr = wrise[k];                              // rising edge of filter s
            if (s > 0) wf = wfall[k];                                   // falling edge of filter s - 1
        }
        float sf;
        memcpy(&sf, &s, 4);
        etab[k] = make_float4(wr * pscale, wf * pscale, sf, 0.f);
    }
}

// CPU model of the tensor-core path for ONE frame of 512 int16 samples: the same butterfly and twiddles, the same operand table
// read through the same layout arithmetic, fp16 products accumulated in fp32, the frame's first sample removed from Y_0 and
// restored in X[0].  d[9][64] = the frame's accumulator columns, block by block, as the epilogue sees them after that correction.
static inline void tcd_host_accumulators(const int16_t* x, float (*d)[64]) {
    static std::vector<__half> b_hi, b_lo;
    static std::vector<float> tw;
    if (b_hi.empty()) { tcd_build_b(b_hi, b_lo); tcd_build_tw(tw); }
    std::vector<float> a((size_t)TCD_BLOCKS * 64);
    for (int g = 0; g < 8; ++g)
        for (int j = 0; j < 4; ++j) {
            const int n2 = 4 * g + j;
            float in[16], yr[9], yi[9], zr[9], zi[9];
            for (int q = 0; q < 16; ++q) in[q] = (float)x[n2 + 32 * q] * TCD_IN_SCALE;
            rdft16_x2(in, yr, yi);
            tcd_twiddle(yr, yi, tw.data() + (size_t)n2 * TCD_TW_STRIDE, TCD_X0_Y * (float)x[0], zr, zi);
            for (int b = 0; b < TCD_BLOCKS; ++b) { a[b * 64 + 8 * g + tcd_kslot(j, 0, g)] = zr[b]; a[b * 64 + 8 * g + tcd_kslot(j, 1, g)] = zi[b]; }
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
                    const float pa = __half2float(pass == 0 ? al : ah), pb = __half2float(pass == 1 ? b_lo[o] : b_hi[o]);
                    acc += pa * pb;
                }
            d[b][n] = acc;
        }
    d[0][0] += TCD_X0_D * (float)x[0];     // the model transforms x - x[0] (exact zeros for constant input) and restores X[0] here
}

// |X[k]|^2 of the raw samples, k = 0..256
static inline void tcd_host_power(const int16_t* x, double* power) {
    float d[TCD_BLOCKS][64];
    tcd_host_accumulators(x, d);
    const double inv = 1.0 / ((double)TCD_A_SCALE * (double)TCD_A_SCALE);
    for (int b = 0; b < TCD_BLOCKS; ++b)
        for (int half = 0; half < 2; ++half)
            for (int m = 0; m < 16; ++m) {
                const int k = tcd_col_bin(b, 32 * half + m);
                if (k < 0) continue;
                const double re = d[b][32 * half + m], im = d[b][32 * half + 16 + m];
                power[k] = (k == 0 || k == 256) ? re * re * inv : (re * re + im * im) * inv;
            }
}

// The epilogue's arithmetic for one frame (fp32): per-segment rising / falling sums in column order, log, DCT, c0.
static inline void tcd_host_epilogue(const float (*d)[64], const float4* etab, const float* dct, int n_filt, int n_out, float pscale,
                                     float* out) {
    float rise[TCD_MAX_FILT + 2] = {0}, fall[TCD_MAX_FILT + 2] = {0}, tot = 0.f;
    for (int b = 0; b < TCD_BLOCKS; ++b)
        for (int half = 0; half < 2; ++half)
            for (int m = 0; m < 16; ++m) {
                const int k = tcd_col_bin(b, 32 * half + m);
                if (k < 0) continue;
                const float re = d[b][32 * half + m], im = d[b][32 * half + 16 + m];
                const float p = (k == 0 || k == 256) ? re * re : fmaf(im, im, re * re);
                int s;
                memcpy(&s, &etab[k].z, 4);
                tot += p;
                rise[s] = fmaf(etab[k].x, p, rise[s]);                  // weights carry pscale here (a power of two: exact)
                fall[s] = fmaf(etab[k].y, p, fall[s]);
            }
    const float eps = 2.220446049250313e-16f;
    float lg[TCD_MAX_FILT];
    for (int j = 0; j < n_filt; ++j) lg[j] = logf(fmaxf(rise[j] + fall[j + 1], eps));
    for (int o = 0; o < n_out; ++o) {
        float v = 0.f;
        for (int j = 0; j < n_filt; ++j) v = fmaf(dct[(size_t)o * 24 + j], lg[j], v);
        out[o] = o == 0 ? logf(fmaxf(tot * pscale, eps)) : v;
    }
}

}  // namespace pb
