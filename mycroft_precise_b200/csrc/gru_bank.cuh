// gru_bank.cuh -- K2 for the fused family of networks (H <= 24, feature_size <= 16, no deltas, any activation pair): the
// default network's large-batch scan, and every such network of a model bank in ONE launch over the handle's shared MFCC ring.
//
// The per-step products run on the warp-level tensor cores in fp16 x 3 (hi / lo split of both operands, fp32 accumulate:
// a_lo b_hi + a_hi b_lo + a_hi b_hi) on mma.sync m16n8k16 / m16n8k8: one k16 + one k8 MMA per n-tile and pass cover the 24
// (padded) hidden units.  Pieces of 11 bits each, 22 bits per product like 3xTF32 (CPU emulation on the default network:
// 7.6e-8 vs 4.7e-8).  Hidden units sit in the k index in natural order (thread t of a quad holds units 8 tile + 2t, 2t + 1 in
// its accumulators = the (2t, 2t + 1) and (2t + 8, 2t + 9) k pairs of the A fragment), so h turns into the next step's A
// operand with two F2FP packs per n-tile and no data movement.
//
// A warp owns a 16-stream tile.  At each of the T steps it loads the tile's MFCC rows once, splits them into fp16 hi / lo A
// fragments once, and then runs, model after model, the x.W products (one k16 MMA per n-tile and pass) and the h.U products
// (mma3_f16).  Each model's h stays in registers, so the M models give the warp M independent dependency chains per step
// while the window's rows are read once per tick for all of them.  Per model the accumulation order is bias, x part, h part.
#pragma once
#include <cuda_fp16.h>

#include "gru_kernels.cuh"

namespace pb {

__device__ __forceinline__ void mma_f16_k16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_f16_k8(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t b0) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a0), "r"(a1), "r"(b0));
}
// (x, y) -> fp16 hi pair and the pair of residuals
__device__ __forceinline__ void split_f16(float x, float y, uint32_t& hi, uint32_t& lo) {
    const __half2 h = __floats2half2_rn(x, y);
    const float2 f = __half22float2(h);
    const __half2 l = __floats2half2_rn(x - f.x, y - f.y);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = *reinterpret_cast<const uint32_t*>(&l);
}
// A fragments of a 24-unit vector held in accumulator layout v[tile][e]: k-tile 0 (units 0..15) as a k16 fragment, units 16..23 as a k8 one
__device__ __forceinline__ void frag_f16(const float (&v)[3][4], uint32_t (&ah)[4], uint32_t (&al)[4], uint32_t (&bh)[2], uint32_t (&bl)[2]) {
    split_f16(v[0][0], v[0][1], ah[0], al[0]);       // row g,     k 2t, 2t + 1
    split_f16(v[0][2], v[0][3], ah[1], al[1]);       // row g + 8
    split_f16(v[1][0], v[1][1], ah[2], al[2]);       // row g,     k 2t + 8, 2t + 9
    split_f16(v[1][2], v[1][3], ah[3], al[3]);
    split_f16(v[2][0], v[2][1], bh[0], bl[0]);       // units 16 + 2t, + 1: the k8 fragment
    split_f16(v[2][2], v[2][3], bh[1], bl[1]);
}
// acc[nt0 .. nt0 + 2] += v . B over the 24 units, three passes
__device__ __forceinline__ void mma3_f16(float (*acc)[4], int nt0, const uint32_t (&ah)[4], const uint32_t (&al)[4], const uint32_t (&ch)[2],
                                         const uint32_t (&cl)[2], const uint4* sB, int lane) {
    uint4 w0[3], w1[3];
#pragma unroll
    for (int q = 0; q < 3; ++q) { w0[q] = sB[(nt0 + q) * 32 + lane]; w1[q] = sB[(MMA_NT + nt0 + q) * 32 + lane]; }
#pragma unroll
    for (int q = 0; q < 3; ++q) { mma_f16_k16(acc[nt0 + q], al, w0[q].x, w0[q].y); mma_f16_k8(acc[nt0 + q], cl[0], cl[1], w1[q].x); }
#pragma unroll
    for (int q = 0; q < 3; ++q) { mma_f16_k16(acc[nt0 + q], ah, w0[q].z, w0[q].w); mma_f16_k8(acc[nt0 + q], ch[0], ch[1], w1[q].z); }
#pragma unroll
    for (int q = 0; q < 3; ++q) { mma_f16_k16(acc[nt0 + q], ah, w0[q].x, w0[q].y); mma_f16_k8(acc[nt0 + q], ch[0], ch[1], w1[q].x); }
}

constexpr int BANK_MAX_MODELS = 8;                                   // PB_MAX_MODELS
constexpr int BANK_MAX_H = 24, BANK_MAX_F = 16;                      // the fused family
// One model in shared memory: recurrent fragments [2][MMA_NT][32] and input fragments [MMA_NT][32] (uint4, as upload_frag16
// builds them: 9 216 + 4 608 B), then bias [3][24] and dense weights [24] as floats.
constexpr int BANK_FRAG_U4 = 3 * MMA_NT * 32;
constexpr int BANK_MODEL_SMEM = BANK_FRAG_U4 * 16 + (72 + 24) * 4;   // 14 208 B

struct BankModelW {
    const uint4* bfrag;              // [2 k-tiles][MMA_NT][32 lanes] (b0_hi, b1_hi, b0_lo, b1_lo) as half2; k-tile 1 uses b0 only (units 16..23)
    const uint4* xfrag;              // [MMA_NT][32 lanes]: the input weights (features 0..15 as one k16 fragment), same packing
    const float* bias;               // [3][24] padded per gate
    const float* wd;                 // [24] padded
    float bd;
    int act, ract;                   // PB_ACT_* / PB_RACT_*
};

struct BankParams {
    BankModelW w[BANK_MAX_MODELS];
    DecodeParams dp[BANK_MAX_MODELS];
    K2Out o[BANK_MAX_MODELS];        // each model's outputs, trigger array and count slot
};

// RING: rows from the stream ring (a tick); otherwise from in.inputs, [n][T][F_base] contiguous (pb_predict).
template <int NM, bool RING>
__global__ void __launch_bounds__(MMA_THREADS, NM == 1 ? 4 : 1)      // NM = 1: 128 registers (ptxas alone picks 96 and spills)
gru_bank_kernel(const __grid_constant__ BankParams P, K2In in, long long n) {
    extern __shared__ __align__(16) unsigned char bank_smem[];
#pragma unroll 1
    for (int m = 0; m < NM; ++m) {
        uint4* sf = reinterpret_cast<uint4*>(bank_smem + m * BANK_MODEL_SMEM);
        float* sb = reinterpret_cast<float*>(sf + BANK_FRAG_U4);
        for (int e = threadIdx.x; e < 2 * MMA_NT * 32; e += blockDim.x) sf[e] = __ldg(P.w[m].bfrag + e);
        for (int e = threadIdx.x; e < MMA_NT * 32; e += blockDim.x) sf[2 * MMA_NT * 32 + e] = __ldg(P.w[m].xfrag + e);
        for (int e = threadIdx.x; e < 72; e += blockDim.x) sb[e] = __ldg(P.w[m].bias + e);
        for (int e = threadIdx.x; e < 24; e += blockDim.x) sb[72 + e] = __ldg(P.w[m].wd + e);
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    const long long base = ((long long)blockIdx.x * (MMA_THREADS / 32) + warp) * 16;
    if (base >= n) return;
    const int F = in.F_base;
    long long idx[2];
    int sid[2];
    RingCursor cur[2];
    bool ok[2];
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
        idx[hf] = base + g + 8 * hf;
        ok[hf] = idx[hf] < n;
        sid[hf] = 0;
        if (RING && ok[hf]) {
            sid[hf] = in.ids ? in.ids[idx[hf]] : (int)idx[hf];
            const long long ns = in.n_samples[sid[hf]];
            cur[hf].init(in, sid[hf], ns >= in.window ? (ns - in.window) / in.hop + 1 : 0);
        }
    }
    float hreg[NM][3][4];
#pragma unroll
    for (int m = 0; m < NM; ++m)
#pragma unroll
        for (int nt = 0; nt < 3; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) hreg[m][nt][e] = 0.f;

#pragma unroll 1
    for (int step = 0; step < in.T; ++step) {
        // ---- the tile's MFCC row as a k16 A fragment: a0 / a1 = rows g / g + 8 at k 2t, 2t + 1; a2 / a3 at k 2t + 8, 2t + 9
        float xv[2][4];
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            const float* row = nullptr;                                     // stays nullptr: a row before the stream's first frame
            if (ok[hf]) row = RING ? cur[hf].next(step) : in.inputs + (idx[hf] * in.T + step) * F;
            xv[hf][0] = (row != nullptr && 2 * t < F) ? __ldg(row + 2 * t) : 0.f;
            xv[hf][1] = (row != nullptr && 2 * t + 1 < F) ? __ldg(row + 2 * t + 1) : 0.f;
            xv[hf][2] = (row != nullptr && 2 * t + 8 < F) ? __ldg(row + 2 * t + 8) : 0.f;
            xv[hf][3] = (row != nullptr && 2 * t + 9 < F) ? __ldg(row + 2 * t + 9) : 0.f;
        }
        uint32_t xh[4], xl[4];
        split_f16(xv[0][0], xv[0][1], xh[0], xl[0]);
        split_f16(xv[1][0], xv[1][1], xh[1], xl[1]);
        split_f16(xv[0][2], xv[0][3], xh[2], xl[2]);
        split_f16(xv[1][2], xv[1][3], xh[3], xl[3]);
#pragma unroll
        for (int m = 0; m < NM; ++m) {
            const uint4* sB = reinterpret_cast<const uint4*>(bank_smem + m * BANK_MODEL_SMEM);
            const uint4* sX = sB + 2 * MMA_NT * 32;
            const float* sBias = reinterpret_cast<const float*>(sB + BANK_FRAG_U4);
            const int ra = P.w[m].ract, ac = P.w[m].act;
            float acc[MMA_NT][4];
#pragma unroll
            for (int nt = 0; nt < MMA_NT; ++nt) {
                const float b0 = sBias[8 * nt + 2 * t], b1 = sBias[8 * nt + 2 * t + 1];
                acc[nt][0] = b0; acc[nt][1] = b1; acc[nt][2] = b0; acc[nt][3] = b1;
            }
            // ---- x part for all three gates (lo.hi, hi.lo, hi.hi)
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
            // ---- h part for z and r
            {
                uint32_t ah[4], al[4], ch[2], cl[2];
                frag_f16(hreg[m], ah, al, ch, cl);
                mma3_f16(acc, 0, ah, al, ch, cl, sB, lane);
                mma3_f16(acc, 3, ah, al, ch, cl, sB, lane);
            }
            // ---- gates; r * h is the A operand of the candidate product
            {
                float rh[3][4];
#pragma unroll
                for (int nt = 0; nt < 3; ++nt)
#pragma unroll
                    for (int e = 0; e < 4; ++e) rh[nt][e] = apply_ract(acc[3 + nt][e], ra) * hreg[m][nt][e];
                uint32_t ah[4], al[4], ch[2], cl[2];
                frag_f16(rh, ah, al, ch, cl);
                mma3_f16(acc, 6, ah, al, ch, cl, sB, lane);
            }
#pragma unroll
            for (int nt = 0; nt < 3; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float z = apply_ract(acc[nt][e], ra);
                    hreg[m][nt][e] = z * hreg[m][nt][e] + (1.f - z) * apply_act(acc[6 + nt][e], ac);
                }
        }
    }
    // ---- per model: Dense(1) (per-thread partial over its 6 units per row, reduced over the quad) and the epilogue
#pragma unroll
    for (int m = 0; m < NM; ++m) {
        const float* sWd = reinterpret_cast<const float*>(bank_smem + m * BANK_MODEL_SMEM + BANK_FRAG_U4 * 16) + 72;
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            float part = 0.f;
#pragma unroll
            for (int nt = 0; nt < 3; ++nt) {
                part = fmaf(hreg[m][nt][2 * hf], sWd[8 * nt + 2 * t], part);
                part = fmaf(hreg[m][nt][2 * hf + 1], sWd[8 * nt + 2 * t + 1], part);
            }
            part += __shfl_xor_sync(0xffffffffu, part, 1);
            part += __shfl_xor_sync(0xffffffffu, part, 2);
            epilogue(part + P.w[m].bd, t == 0 && ok[hf], idx[hf], sid[hf], P.dp[m], P.o[m]);
        }
    }
}

}  // namespace pb
