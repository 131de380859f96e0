// wgmma_probe.cu -- does warpgroup MMA pay for the default window scan, and does it add exactly as mma.sync does?
//
// Throughput / latency: the per-step arithmetic of the default network's scan (H = 24 padded, 16 features, fp16 x 3, Keras
// activations) with the window rows taken from a shared-memory table instead of the ring, in two forms over the same weights:
//   (a) mma.sync: a warp per 16 streams, 54 m16n8k16 + 27 m16n8k8 per step, as bank_scan issues them;
//   (b) wgmma: a warpgroup per 64 streams, 3 x (m64n48k16 + m64n24k16) (x.W for z, r and for the candidate), 6 x m64n48k16
//       (h.U for z, r) and 6 x m64n24k16 (candidate), units 16..23 as a k16 whose upper 8 k-slots are zero.  x.W is not one
//       m64n72k16 per pass: an n24 accumulator inside an n72 one makes ptxas serialize every wgmma of the step (C7511).
//   (c) the 18 wgmma of (b) with fixed operands and nothing between them: the tensor pipe's rate for that instruction mix.
// Each runs at 4 resident CTAs of 128 threads per SM (one full wave) for the rate, and one CTA per SM for the latency.  The
// final h of (a) and (b) must be bit-identical.
// Bit equality: per case, one fp32 accumulator taken from a random start through the six products of mma3_f16 (lo.hi, hi.lo,
// hi.hi over units 0..15 as k16 and units 16..23 as k8) on mma.sync, and the same products in the same order on wgmma.
// Operands are fp16 hi / lo pieces of N(0, s) values: mixed scales, exact cancellation, saturated +-65504 pieces.
//
// nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o wgmma_probe scripts/wgmma_probe.cu; prints one JSON line.
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <vector>

#include "../mycroft_precise_b200/csrc/gru_wg.cuh"

using namespace pb;

#define CKX(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

constexpr int XT = 8;                                    // window rows cycle through XT steps of the table
constexpr int XTAB = XT * 64 * 16;                       // floats: [step][stream][feature]
constexpr int FRAG_BYTES = 3 * MMA_NT * 32 * 16;         // bank_scan's fragment layout (13 824 B)
constexpr int WG_BYTES = 6 * WG_TILE_BYTES;              // X hi, X lo, U0 hi, U0 lo, U1 hi, U1 lo (13 824 B)
constexpr int SCAN_SMEM = XTAB * 4 + 13824 + 72 * 4;

struct ScanArgs {
    const uint4* frag;        // [3][MMA_NT][32]
    const uint8_t* wg;        // WG_BYTES
    const float* bias;        // [72]
    const float* xtab;        // XTAB
    float* hout;              // [ctas * 64][24]
    long long* cycles;        // [ctas]
    int T;
};

__device__ __forceinline__ void load_common(const ScanArgs& a, unsigned char* sm, const void* w, int wbytes) {
    for (int i = threadIdx.x; i < XTAB / 4; i += blockDim.x) reinterpret_cast<float4*>(sm)[i] = reinterpret_cast<const float4*>(a.xtab)[i];
    for (int i = threadIdx.x; i < wbytes / 16; i += blockDim.x) reinterpret_cast<uint4*>(sm + XTAB * 4)[i] = reinterpret_cast<const uint4*>(w)[i];
    for (int i = threadIdx.x; i < 72; i += blockDim.x) reinterpret_cast<float*>(sm + XTAB * 4 + 13824)[i] = a.bias[i];
}

__device__ __forceinline__ void x_rows(const float* xs, int warp, int g, int t, uint32_t (&xh)[4], uint32_t (&xl)[4]) {
    float xv[2][4];
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
        const float* row = xs + (16 * warp + g + 8 * hf) * 16;
        const float2 lo = *reinterpret_cast<const float2*>(row + 2 * t), hi = *reinterpret_cast<const float2*>(row + 2 * t + 8);
        xv[hf][0] = lo.x; xv[hf][1] = lo.y; xv[hf][2] = hi.x; xv[hf][3] = hi.y;
    }
    split_f16(xv[0][0], xv[0][1], xh[0], xl[0]);
    split_f16(xv[1][0], xv[1][1], xh[1], xl[1]);
    split_f16(xv[0][2], xv[0][3], xh[2], xl[2]);
    split_f16(xv[1][2], xv[1][3], xh[3], xl[3]);
}

__device__ __forceinline__ void store_h(const ScanArgs& a, const float (&h)[3][4], int warp, int g, int t) {
    const long long s0 = (long long)blockIdx.x * 64 + 16 * warp + g;
#pragma unroll
    for (int nt = 0; nt < 3; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) a.hout[(s0 + 8 * (e >> 1)) * 24 + 8 * nt + 2 * t + (e & 1)] = h[nt][e];
}

// (a) the mma.sync step sequence of bank_scan<1, true, true>
__global__ void __launch_bounds__(128, 4) scan_mma_kernel(const ScanArgs a) {
    extern __shared__ __align__(16) unsigned char sm[];
    load_common(a, sm, a.frag, FRAG_BYTES);
    __syncthreads();
    const long long c0 = clock64();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    const uint4* sB = reinterpret_cast<const uint4*>(sm + XTAB * 4);
    const uint4* sX = sB + 2 * MMA_NT * 32;
    const float* sBias = reinterpret_cast<const float*>(sm + XTAB * 4 + 13824);
    float h[3][4] = {};
#pragma unroll 1
    for (int step = 0; step < a.T; ++step) {
        uint32_t xh[4], xl[4];
        x_rows(reinterpret_cast<const float*>(sm) + (step & (XT - 1)) * 64 * 16, warp, g, t, xh, xl);
        float acc[MMA_NT][4];
#pragma unroll
        for (int nt = 0; nt < MMA_NT; ++nt) {
            const float b0 = sBias[8 * nt + 2 * t], b1 = sBias[8 * nt + 2 * t + 1];
            acc[nt][0] = b0; acc[nt][1] = b1; acc[nt][2] = b0; acc[nt][3] = b1;
        }
#pragma unroll
        for (int ng = 0; ng < MMA_NT; ng += 3) {
            uint4 w[3];
#pragma unroll
            for (int q = 0; q < 3; ++q) w[q] = sX[(ng + q) * 32 + lane];
#pragma unroll
            for (int q = 0; q < 3; ++q) mma_f16_k16(acc[ng + q], xl, w[q].x, w[q].y);
#pragma unroll
            for (int q = 0; q < 3; ++q) mma_f16_k16(acc[ng + q], xh, w[q].z, w[q].w);
#pragma unroll
            for (int q = 0; q < 3; ++q) mma_f16_k16(acc[ng + q], xh, w[q].x, w[q].y);
        }
        {
            uint32_t ah[4], al[4], ch[2], cl[2];
            frag_f16(h, ah, al, ch, cl);
            mma3_f16(acc, 0, ah, al, ch, cl, sB, lane);
            mma3_f16(acc, 3, ah, al, ch, cl, sB, lane);
        }
        {
            float rh[3][4];
#pragma unroll
            for (int nt = 0; nt < 3; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) rh[nt][e] = __fmul_rn(hard_sigmoid(acc[3 + nt][e]), h[nt][e]);
            uint32_t ah[4], al[4], ch[2], cl[2];
            frag_f16(rh, ah, al, ch, cl);
            mma3_f16(acc, 6, ah, al, ch, cl, sB, lane);
        }
#pragma unroll
        for (int nt = 0; nt < 3; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float z = hard_sigmoid(acc[nt][e]);
                h[nt][e] = __fmaf_rn(z, h[nt][e], __fmul_rn(__fsub_rn(1.f, z), acc[6 + nt][e]));
            }
    }
    const long long c1 = clock64();
    if (threadIdx.x == 0) a.cycles[blockIdx.x] = c1 - c0;
    store_h(a, h, warp, g, t);
}

// (b) the wgmma step sequence
__global__ void __launch_bounds__(128, 4) scan_wg_kernel(const ScanArgs a) {
    extern __shared__ __align__(16) unsigned char sm[];
    load_common(a, sm, a.wg, WG_BYTES);
    wg_fence_smem();
    __syncthreads();
    const long long c0 = clock64();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    const unsigned char* sW = sm + XTAB * 4;
    const float* sBias = reinterpret_cast<const float*>(sm + XTAB * 4 + 13824);
    const uint64_t dXh = wg_desc(sW), dXl = wg_desc(sW + WG_TILE_BYTES), dU0h = wg_desc(sW + 2 * WG_TILE_BYTES),
                   dU0l = wg_desc(sW + 3 * WG_TILE_BYTES), dU1h = wg_desc(sW + 4 * WG_TILE_BYTES), dU1l = wg_desc(sW + 5 * WG_TILE_BYTES);
    constexpr uint64_t C6 = (6 * 256) >> 4;                  // candidate columns start at n-tile 6
    float h[3][4] = {};
#pragma unroll 1
    for (int step = 0; step < a.T; ++step) {
        uint32_t xh[4], xl[4];
        x_rows(reinterpret_cast<const float*>(sm) + (step & (XT - 1)) * 64 * 16, warp, g, t, xh, xl);
        float acc[36];
#pragma unroll
        for (int nt = 0; nt < MMA_NT; ++nt) {
            const float b0 = sBias[8 * nt + 2 * t], b1 = sBias[8 * nt + 2 * t + 1];
            acc[4 * nt] = b0; acc[4 * nt + 1] = b1; acc[4 * nt + 2] = b0; acc[4 * nt + 3] = b1;
        }
        uint32_t ah[4], al[4], ch[4] = {0, 0, 0, 0}, cl[4] = {0, 0, 0, 0};
        {
            uint32_t c2h[2], c2l[2];
            frag_f16(h, ah, al, c2h, c2l);
            ch[0] = c2h[0]; ch[1] = c2h[1]; cl[0] = c2l[0]; cl[1] = c2l[1];
        }
        wg_fence_regs<36>(acc);
        wg_fence();
        wgmma_n48(acc, xl, dXh);
        wgmma_n24(acc + 24, xl, dXh + C6);
        wgmma_n48(acc, xh, dXl);
        wgmma_n24(acc + 24, xh, dXl + C6);
        wgmma_n48(acc, xh, dXh);
        wgmma_n24(acc + 24, xh, dXh + C6);
        wgmma_n48(acc, al, dU0h);
        wgmma_n48(acc, cl, dU1h);
        wgmma_n48(acc, ah, dU0l);
        wgmma_n48(acc, ch, dU1l);
        wgmma_n48(acc, ah, dU0h);
        wgmma_n48(acc, ch, dU1h);
        wg_commit();
        wg_wait<0>();
        wg_fence_regs<36>(acc);
        {
            float rh[3][4];
#pragma unroll
            for (int nt = 0; nt < 3; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) rh[nt][e] = __fmul_rn(hard_sigmoid(acc[4 * (3 + nt) + e]), h[nt][e]);
            uint32_t c2h[2], c2l[2];
            frag_f16(rh, ah, al, c2h, c2l);
            ch[0] = c2h[0]; ch[1] = c2h[1]; cl[0] = c2l[0]; cl[1] = c2l[1];
        }
        wg_fence_regs<12>(acc + 24);
        wg_fence();
        wgmma_n24(acc + 24, al, dU0h + C6);
        wgmma_n24(acc + 24, cl, dU1h + C6);
        wgmma_n24(acc + 24, ah, dU0l + C6);
        wgmma_n24(acc + 24, ch, dU1l + C6);
        wgmma_n24(acc + 24, ah, dU0h + C6);
        wgmma_n24(acc + 24, ch, dU1h + C6);
        wg_commit();
        wg_wait<0>();
        wg_fence_regs<12>(acc + 24);
#pragma unroll
        for (int nt = 0; nt < 3; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float z = hard_sigmoid(acc[4 * nt + e]);
                h[nt][e] = __fmaf_rn(z, h[nt][e], __fmul_rn(__fsub_rn(1.f, z), acc[4 * (6 + nt) + e]));
            }
    }
    const long long c1 = clock64();
    if (threadIdx.x == 0) a.cycles[blockIdx.x] = c1 - c0;
    store_h(a, h, warp, g, t);
}

// (c) the 18 wgmma of (b) per step with fixed A operands, one commit / wait per step and no arithmetic between them: what
// the tensor pipe gives this instruction mix when nothing else is in the way.  Its h is a checksum, not a scan.
__global__ void __launch_bounds__(128, 4) pipe_wg_kernel(const ScanArgs a) {
    extern __shared__ __align__(16) unsigned char sm[];
    load_common(a, sm, a.wg, WG_BYTES);
    wg_fence_smem();
    __syncthreads();
    const long long c0 = clock64();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    const unsigned char* sW = sm + XTAB * 4;
    const float* sBias = reinterpret_cast<const float*>(sm + XTAB * 4 + 13824);
    const uint64_t dXh = wg_desc(sW), dXl = wg_desc(sW + WG_TILE_BYTES), dU0h = wg_desc(sW + 2 * WG_TILE_BYTES),
                   dU0l = wg_desc(sW + 3 * WG_TILE_BYTES), dU1h = wg_desc(sW + 4 * WG_TILE_BYTES), dU1l = wg_desc(sW + 5 * WG_TILE_BYTES);
    constexpr uint64_t C6 = (6 * 256) >> 4;
    uint32_t xh[4], xl[4];
    x_rows(reinterpret_cast<const float*>(sm), warp, g, t, xh, xl);
    float h[3][4] = {};
#pragma unroll 1
    for (int step = 0; step < a.T; ++step) {
        float acc[36];
#pragma unroll
        for (int nt = 0; nt < MMA_NT; ++nt) {
            const float b0 = sBias[8 * nt + 2 * t], b1 = sBias[8 * nt + 2 * t + 1];
            acc[4 * nt] = b0; acc[4 * nt + 1] = b1; acc[4 * nt + 2] = b0; acc[4 * nt + 3] = b1;
        }
        wg_fence_regs<36>(acc);
        wg_fence();
        wgmma_n48(acc, xl, dXh);
        wgmma_n24(acc + 24, xl, dXh + C6);
        wgmma_n48(acc, xh, dXl);
        wgmma_n24(acc + 24, xh, dXl + C6);
        wgmma_n48(acc, xh, dXh);
        wgmma_n24(acc + 24, xh, dXh + C6);
        wgmma_n48(acc, xl, dU0h);
        wgmma_n48(acc, xh, dU1h);
        wgmma_n48(acc, xl, dU0l);
        wgmma_n48(acc, xh, dU1l);
        wgmma_n48(acc, xl, dU0h);
        wgmma_n48(acc, xh, dU1h);
        wgmma_n24(acc + 24, xl, dU0h + C6);
        wgmma_n24(acc + 24, xh, dU1h + C6);
        wgmma_n24(acc + 24, xl, dU0l + C6);
        wgmma_n24(acc + 24, xh, dU1l + C6);
        wgmma_n24(acc + 24, xl, dU0h + C6);
        wgmma_n24(acc + 24, xh, dU1h + C6);
        wg_commit();
        wg_wait<0>();
        wg_fence_regs<36>(acc);
#pragma unroll
        for (int nt = 0; nt < 3; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) h[nt][e] += acc[4 * nt + e] + acc[4 * (3 + nt) + e] + acc[4 * (6 + nt) + e];
    }
    const long long c1 = clock64();
    if (threadIdx.x == 0) a.cycles[blockIdx.x] = c1 - c0;
    store_h(a, h, warp, g, t);
}

// ---- bit equality of single accumulators
__device__ __forceinline__ uint64_t mix64(uint64_t x) {
    x += 0x9e3779b97f4a7c15ull;
    x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
    x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
    return x ^ (x >> 31);
}
// N(0, 1) (Box-Muller) scaled by mode: 0 plain (scale per case), 1 plain (paired for cancellation by the caller),
// 2 values near and beyond the fp16 range (saturated pieces), 3 per-element scale 2^-20 .. 2^15
__device__ __forceinline__ float draw(uint64_t key, int mode, float case_scale) {
    const uint64_t r = mix64(key);
    const float u1 = ((uint32_t)r + 1.f) * 2.3283064e-10f, u2 = (uint32_t)(r >> 32) * 2.3283064e-10f;
    float v = sqrtf(-2.f * logf(u1)) * cospif(2.f * u2);
    const uint32_t s = (uint32_t)mix64(key ^ 0x5bd1e995ull);
    if (mode == 2) v *= (s & 3) == 0 ? 2e5f : (s & 3) == 1 ? 65504.f : 6e4f;
    else if (mode == 3) v = ldexpf(v, (int)(s % 36) - 20);
    else v *= case_scale;
    return v;
}
__device__ __forceinline__ uint16_t f16_bits(float v) { const __half h = __float2half_rn(v); uint16_t u; memcpy(&u, &h, 2); return u; }
__device__ __forceinline__ uint16_t sat16(float v) { return f16_bits(fminf(fmaxf(v, -65504.f), 65504.f)); }

// One warpgroup per CTA.  Per iteration: B = 24 (k) x 24 (n) values split in hi / lo tiles (k 0..15 = tile 0, k 16..23 =
// tile 1 with zero k-slots 8..15), A = 64 x 24 values split likewise, C = 64 x 24 start values.  counts[0] += cases,
// counts[1] += mismatches; the first mismatch goes to bad[0..3] (mma bits, wgmma bits, iteration, mode).
__global__ void __launch_bounds__(128) eq_kernel(uint64_t seed, int iters, unsigned long long* counts, unsigned* bad) {
    __shared__ __align__(128) unsigned char sT[4 * 768];      // tile 0 hi, tile 0 lo, tile 1 hi, tile 1 lo; 24 columns each
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    unsigned long long miss = 0;
    for (int it = 0; it < iters; ++it) {
        const uint64_t cs = mix64(seed ^ ((uint64_t)blockIdx.x << 32) ^ (uint64_t)it);
        const int mode = (int)(cs & 3);
        const float sa = ldexpf(1.f, (int)((cs >> 8) % 24) - 12), sb = ldexpf(1.f, (int)((cs >> 16) % 24) - 12);
        const float sc = (cs >> 24) & 1 ? 0.f : ldexpf(1.f, (int)((cs >> 32) % 24) - 8);
        auto bval = [&](int k, int n) {                       // mode 1: k 8..15 (and 20..23) cancel k 0..7 (16..19)
            const int kk = mode == 1 && ((k & 15) >= 8 || k >= 20) ? (k >= 16 ? k - 4 : k - 8) : k;
            const float v = draw(cs ^ (0x1000ull + kk * 64 + n), mode, sb);
            return kk != k ? -v : v;
        };
        auto aval = [&](int m, int k) {
            const int kk = mode == 1 && ((k & 15) >= 8 || k >= 20) ? (k >= 16 ? k - 4 : k - 8) : k;
            return draw(cs ^ (0x100000ull + (uint64_t)m * 64 + kk), mode, sa);
        };
        __syncthreads();
        for (int i = threadIdx.x; i < 2 * 16 * 24; i += blockDim.x) {
            const int kt = i / (16 * 24), k = (i / 24) % 16, n = i % 24;
            const bool real = kt == 0 || k < 8;
            const float v = real ? bval(16 * kt + k, n) : 0.f;
            const uint16_t hi = sat16(v), lo = sat16(v - __half2float(*reinterpret_cast<const __half*>(&hi)));
            *reinterpret_cast<uint16_t*>(sT + (2 * kt) * 768 + wg_b_offset(k, n)) = hi;
            *reinterpret_cast<uint16_t*>(sT + (2 * kt + 1) * 768 + wg_b_offset(k, n)) = lo;
        }
        wg_fence_smem();
        __syncthreads();
        // A pieces in mma.m16n8k16 A layout: v[nt][e] = A(row g + 8 (e >> 1), k 8 nt + 2 t + (e & 1))
        float av[3][4];
        const int r0 = 16 * warp + g;
#pragma unroll
        for (int kt = 0; kt < 3; ++kt)
#pragma unroll
            for (int e = 0; e < 4; ++e) av[kt][e] = aval(r0 + 8 * (e >> 1), 8 * kt + 2 * t + (e & 1));
        uint32_t ah[4], al[4], ch2[2], cl2[2];
        frag_f16(av, ah, al, ch2, cl2);
        float c[12], dm[12], dw[12];
#pragma unroll
        for (int j = 0; j < 3; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) c[4 * j + e] = draw(cs ^ (0x7000000ull + (uint64_t)(r0 + 8 * (e >> 1)) * 64 + 8 * j + 2 * t + (e & 1)), 0, sc);
        // mma.sync, in mma3_f16's order
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            float d[4] = {c[4 * j], c[4 * j + 1], c[4 * j + 2], c[4 * j + 3]};
            auto ld = [&](int tile, int k) { return *reinterpret_cast<const uint32_t*>(sT + tile * 768 + wg_b_offset(k, 8 * j + g)); };
            mma_f16_k16(d, al, ld(0, 2 * t), ld(0, 2 * t + 8));
            mma_f16_k8(d, cl2[0], cl2[1], ld(2, 2 * t));
            mma_f16_k16(d, ah, ld(1, 2 * t), ld(1, 2 * t + 8));
            mma_f16_k8(d, ch2[0], ch2[1], ld(3, 2 * t));
            mma_f16_k16(d, ah, ld(0, 2 * t), ld(0, 2 * t + 8));
            mma_f16_k8(d, ch2[0], ch2[1], ld(2, 2 * t));
#pragma unroll
            for (int e = 0; e < 4; ++e) dm[4 * j + e] = d[e];
        }
        // wgmma, the same products
        const uint32_t ch[4] = {ch2[0], ch2[1], 0u, 0u}, cl[4] = {cl2[0], cl2[1], 0u, 0u};
#pragma unroll
        for (int i = 0; i < 12; ++i) dw[i] = c[i];
        wg_fence();
        wgmma_n24(dw, al, wg_desc(sT));
        wgmma_n24(dw, cl, wg_desc(sT + 2 * 768));
        wgmma_n24(dw, ah, wg_desc(sT + 768));
        wgmma_n24(dw, ch, wg_desc(sT + 3 * 768));
        wgmma_n24(dw, ah, wg_desc(sT));
        wgmma_n24(dw, ch, wg_desc(sT + 2 * 768));
        wg_commit();
        wg_wait<0>();
        wg_fence_regs<12>(dw);
#pragma unroll
        for (int i = 0; i < 12; ++i) {
            const unsigned um = __float_as_uint(dm[i]), uw = __float_as_uint(dw[i]);
            if (um != uw) {
                ++miss;
                if (atomicCAS(bad + 4, 0u, 1u) == 0u) { bad[0] = um; bad[1] = uw; bad[2] = it; bad[3] = mode; }
            }
        }
    }
    atomicAdd(counts + 1, miss);
    if (threadIdx.x == 0) atomicAdd(counts, (unsigned long long)iters * 64 * 24);
}

// ---- host
static uint16_t h16(float v) { const __half h = __float2half_rn(v); uint16_t u; memcpy(&u, &h, 2); return u; }
static float f16(uint16_t u) { __half h; memcpy(&h, &u, 2); return __half2float(h); }

int main(int argc, char** argv) {
    const int T = argc > 1 ? atoi(argv[1]) : 4096;
    const int eq_iters = argc > 2 ? atoi(argv[2]) : 24;
    int dev = 0, sms = 0, clk = 0;
    CKX(cudaSetDevice(dev));
    cudaDeviceProp prop;
    CKX(cudaGetDeviceProperties(&prop, dev));
    CKX(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    CKX(cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, dev));

    // weights: H = 24 fully populated, 16 features, N(0, 0.3); bias N(0, 0.1); rows N(0, 4)
    std::mt19937 rng(1234);
    std::normal_distribution<float> nd(0.f, 1.f);
    std::vector<float> W(16 * 72), U(24 * 72), bias(72), xtab(XTAB);
    for (auto& v : W) v = 0.3f * nd(rng);
    for (auto& v : U) v = 0.3f * nd(rng);
    for (auto& v : bias) v = 0.1f * nd(rng);
    for (auto& v : xtab) v = 4.f * nd(rng);
    auto hi = [](float v) { return h16(v); };
    auto lo = [](float v) { return h16(v - f16(h16(v))); };
    auto pk = [](uint16_t a, uint16_t b) { return (uint32_t)a | ((uint32_t)b << 16); };
    // bank_scan fragments, as build_frag16 packs them: column n = 8 nt + g, k rows 2t, 2t + 1 (b0) and 2t + 8, 2t + 9 (b1)
    std::vector<uint4> frag(3 * MMA_NT * 32);
    auto ukt = [&](int kt, int k, int n) { const int u = 16 * kt + k; return (kt == 1 && k >= 8) ? 0.f : U[u * 72 + n]; };
    for (int kt = 0; kt < 3; ++kt)
        for (int nt = 0; nt < MMA_NT; ++nt)
            for (int lane = 0; lane < 32; ++lane) {
                const int g = lane >> 2, t = lane & 3, n = 8 * nt + g;
                auto v = [&](int k) { return kt < 2 ? ukt(kt, k, n) : W[k * 72 + n]; };
                frag[(kt * MMA_NT + nt) * 32 + lane] = make_uint4(pk(hi(v(2 * t)), hi(v(2 * t + 1))), pk(hi(v(2 * t + 8)), hi(v(2 * t + 9))),
                                                                  pk(lo(v(2 * t)), lo(v(2 * t + 1))), pk(lo(v(2 * t + 8)), lo(v(2 * t + 9))));
            }
    // wgmma tiles
    std::vector<uint8_t> wg(WG_BYTES, 0);
    auto put = [&](int tile, int k, int n, uint16_t b) { memcpy(&wg[tile * WG_TILE_BYTES + wg_b_offset(k, n)], &b, 2); };
    for (int k = 0; k < 16; ++k)
        for (int n = 0; n < 72; ++n) {
            put(0, k, n, hi(W[k * 72 + n])); put(1, k, n, lo(W[k * 72 + n]));
            put(2, k, n, hi(ukt(0, k, n))); put(3, k, n, lo(ukt(0, k, n)));
            put(4, k, n, hi(ukt(1, k, n))); put(5, k, n, lo(ukt(1, k, n)));
        }

    uint4* d_frag; uint8_t* d_wg; float *d_bias, *d_x, *d_h[3]; long long* d_cyc;
    const int ctas = sms * 4;
    CKX(cudaMalloc(&d_frag, frag.size() * 16));
    CKX(cudaMalloc(&d_wg, wg.size()));
    CKX(cudaMalloc(&d_bias, 72 * 4));
    CKX(cudaMalloc(&d_x, XTAB * 4));
    for (int i = 0; i < 3; ++i) CKX(cudaMalloc(&d_h[i], (size_t)ctas * 64 * 24 * 4));
    CKX(cudaMalloc(&d_cyc, ctas * 8));
    CKX(cudaMemcpy(d_frag, frag.data(), frag.size() * 16, cudaMemcpyHostToDevice));
    CKX(cudaMemcpy(d_wg, wg.data(), wg.size(), cudaMemcpyHostToDevice));
    CKX(cudaMemcpy(d_bias, bias.data(), 72 * 4, cudaMemcpyHostToDevice));
    CKX(cudaMemcpy(d_x, xtab.data(), XTAB * 4, cudaMemcpyHostToDevice));
    CKX(cudaFuncSetAttribute(scan_mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SCAN_SMEM));
    CKX(cudaFuncSetAttribute(scan_wg_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SCAN_SMEM));
    CKX(cudaFuncSetAttribute(pipe_wg_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SCAN_SMEM));
    int occ[3];
    CKX(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ[0], scan_mma_kernel, 128, SCAN_SMEM));
    CKX(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ[1], scan_wg_kernel, 128, SCAN_SMEM));
    CKX(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ[2], pipe_wg_kernel, 128, SCAN_SMEM));

    cudaEvent_t e0, e1;
    CKX(cudaEventCreate(&e0)); CKX(cudaEventCreate(&e1));
    // rate: ms for one wave of `grid` CTAs, best of 5 after a warm-up; latency: cycles per step of one CTA per SM
    auto run = [&](int which, int grid, double& best_ms, double& cyc_per_step) {
        ScanArgs a{d_frag, d_wg, d_bias, d_x, d_h[which], d_cyc, T};
        best_ms = 1e30;
        for (int r = 0; r < 6; ++r) {
            CKX(cudaEventRecord(e0));
            if (which == 0) scan_mma_kernel<<<grid, 128, SCAN_SMEM>>>(a);
            else if (which == 1) scan_wg_kernel<<<grid, 128, SCAN_SMEM>>>(a);
            else pipe_wg_kernel<<<grid, 128, SCAN_SMEM>>>(a);
            CKX(cudaEventRecord(e1));
            CKX(cudaEventSynchronize(e1));
            CKX(cudaGetLastError());
            float ms; CKX(cudaEventElapsedTime(&ms, e0, e1));
            if (r > 0) best_ms = std::min(best_ms, (double)ms);
        }
        std::vector<long long> cyc(grid);
        CKX(cudaMemcpy(cyc.data(), d_cyc, grid * 8, cudaMemcpyDeviceToHost));
        std::sort(cyc.begin(), cyc.end());
        cyc_per_step = (double)cyc[grid / 2] / T;
    };
    double ms[3][2], cps[3][2];
    for (int w = 0; w < 3; ++w) {
        run(w, sms, ms[w][1], cps[w][1]);            // latency: one CTA per SM
        run(w, ctas, ms[w][0], cps[w][0]);           // rate: four CTAs per SM (outputs kept for the comparison)
    }
    std::vector<float> hm((size_t)ctas * 64 * 24), hw(hm.size());
    CKX(cudaMemcpy(hm.data(), d_h[0], hm.size() * 4, cudaMemcpyDeviceToHost));
    CKX(cudaMemcpy(hw.data(), d_h[1], hw.size() * 4, cudaMemcpyDeviceToHost));
    long long scan_diff = 0;
    for (size_t i = 0; i < hm.size(); ++i) scan_diff += memcmp(&hm[i], &hw[i], 4) != 0;
    bool finite = true;
    for (float v : hm) finite = finite && std::isfinite(v);

    unsigned long long* d_cnt; unsigned* d_bad;
    CKX(cudaMalloc(&d_cnt, 16)); CKX(cudaMalloc(&d_bad, 20));
    CKX(cudaMemset(d_cnt, 0, 16)); CKX(cudaMemset(d_bad, 0, 20));
    CKX(cudaEventRecord(e0));
    eq_kernel<<<ctas * 8, 128>>>(0x243f6a8885a308d3ull, eq_iters, d_cnt, d_bad);
    CKX(cudaEventRecord(e1));
    CKX(cudaEventSynchronize(e1));
    CKX(cudaGetLastError());
    unsigned long long cnt[2]; unsigned bad[5];
    CKX(cudaMemcpy(cnt, d_cnt, 16, cudaMemcpyDeviceToHost));
    CKX(cudaMemcpy(bad, d_bad, 20, cudaMemcpyDeviceToHost));

    const double ss_a = (double)ctas * 64 * T / (ms[0][0] * 1e-3), ss_b = (double)ctas * 64 * T / (ms[1][0] * 1e-3),
                 ss_c = (double)ctas * 64 * T / (ms[2][0] * 1e-3);
    const char* form = "{\"stream_steps_per_s\": %.4e, \"wave_ms\": %.4f, \"cycles_per_step_4cta\": %.1f, "
                       "\"latency_cycles_per_step_1cta\": %.1f, \"latency_us_per_step_1cta\": %.4f}";
    printf("{\"card\": \"%s\", \"sms\": %d, \"sm_clock_max_mhz\": %d, \"steps\": %d, \"occupancy_ctas_per_sm\": [%d, %d, %d]",
           prop.name, sms, clk / 1000, T, occ[0], occ[1], occ[2]);
    const char* names[3] = {"mma_sync", "wgmma", "wgmma_pipe_only"};
    for (int w = 0; w < 3; ++w) {
        printf(", \"%s\": ", names[w]);
        printf(form, (double)ctas * 64 * T / (ms[w][0] * 1e-3), ms[w][0], cps[w][0], cps[w][1], ms[w][1] * 1e3 / T);
    }
    printf(", \"wgmma_over_mma_sync\": %.3f, \"pipe_only_over_mma_sync\": %.3f, \"scan_h_values\": %zu, "
           "\"scan_h_bit_differences\": %lld, \"scan_h_finite\": %s, \"eq_cases\": %llu, \"eq_mismatches\": %llu, "
           "\"eq_first_mismatch\": [%u, %u, %u, %u]}\n",
           ss_b / ss_a, ss_c / ss_a, hm.size(), scan_diff, finite ? "true" : "false", cnt[0], cnt[1], bad[0], bad[1], bad[2], bad[3]);
    return 0;
}
