// gru_wide.cuh -- K2 for the other networks (H <= 128, F <= 40; BASELINE configs[2]) on mma.sync.m16n8k8 TF32 with the 3xTF32
// split, same recurrence as gru_tiled_kernel.  A CTA owns 128 streams; warp w owns hidden units 16 w .. 16 w + 15 (its z, r
// and candidate columns), so each pre-split weight fragment is read from L2 once per CTA, step and M half.  [x | h], r h
// and z are fp32 rows in shared memory (stride 4 mod 32 words: conflict-free A fragment loads).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "gru_kernels.cuh"

namespace pb {

constexpr int WG_THREADS = 256;
constexpr int WG_STREAMS = 128;
constexpr int WG_MAX_H = 128;
constexpr int WG_MAX_F = 40;

struct GruWideW {
    const uint4* b1;     // phase 1 fragments [kstep][ntile: z units HP / 8, then r units HP / 8][lane]: (b0 hi, b1 hi, b0 lo, b1 lo)
    const uint4* b2;     // phase 2 (candidate) fragments [kstep][ntile HP / 8][lane]
    const float* bias;   // [3 HP]: z, r, candidate (zero padded)
    const float* wd;     // [H]
    float bd;
    int H, F, FP, HP;    // FP = F rounded up to 8, HP = H rounded up to 16
    int act, ract;
};

__host__ __device__ constexpr int wg_as(int FP, int HP) { return FP + HP + 4; }   // floats per row of [x | h]
__host__ __device__ constexpr int wg_rs(int HP) { return HP + 4; }                 // floats per row of r h and of z
__host__ __device__ constexpr size_t wg_smem(int FP, int HP) { return (size_t)WG_STREAMS * (wg_as(FP, HP) + 2 * wg_rs(HP)) * sizeof(float); }

__device__ __forceinline__ void wg_afrag(const float* base, int stride, int row, int k, uint32_t (&hi)[4], uint32_t (&lo)[4]) {
    float v[4];
    v[0] = base[row * stride + k];           v[1] = base[(row + 8) * stride + k];
    v[2] = base[row * stride + k + 4];       v[3] = base[(row + 8) * stride + k + 4];
    split_tf32(v, hi, lo);
}

// The scan of one tile: items base .. base + 127 (those below n) of `in`, base = tile_base(), network W, Dense and epilogue
// into out.  Shared by gru_wide_kernel (W a kernel parameter, one tile per CTA) and gru_wide_rows_kernel (rows.cuh: W from a
// per-network table).  tile_base is called where the kernel always computed its base, which keeps gru_wide_kernel's SASS.
// PIN_FMA: the state update z h + (1 - z) a with gru_wide_kernel's contractions spelled out (see below), for kernels that
// must reproduce its bits; gru_wide_kernel itself leaves the choice to the compiler.
template <bool RING, bool PIN_FMA, typename TileBase>
__device__ __forceinline__ void gru_wide_tile(const GruWideW& W, const K2In& in, TileBase tile_base, long long n, const DecodeParams& dp,
                                              const K2Out& out) {
    extern __shared__ __align__(16) float wg_sm[];
    const int F = W.F, H = W.H, FP = W.FP, HP = W.HP;
    const int AS = wg_as(FP, HP), RS = wg_rs(HP);
    float* A = wg_sm;                              // [128][AS]: x_t in [0, F), h in [FP, FP + H)
    float* RH = A + WG_STREAMS * AS;               // [128][RS]: r h
    float* Z = RH + WG_STREAMS * RS;               // [128][RS]: z
    __shared__ int s_sid[WG_STREAMS];
    __shared__ long long s_rel[WG_STREAMS];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
    const long long base = tile_base();
    if (tid < WG_STREAMS) {
        const long long i = base + tid;
        int sid = 0; long long rel = 0;
        if (RING && i < n) {
            sid = in.ids ? in.ids[i] : (int)i;
            const long long ns = in.n_samples[sid];
            rel = ns >= in.window ? (ns - in.window) / in.hop + 1 : 0;
        }
        s_sid[tid] = sid; s_rel[tid] = rel;
    }
    for (int e = tid; e < WG_STREAMS * AS; e += WG_THREADS) A[e] = 0.f;
    __syncthreads();
    const int KX = FP / 8, KS = KX + HP / 8, NT1 = HP / 4, NT2 = HP / 8;
    const bool active = warp < HP / 16;            // warps beyond the padded width only stage inputs
    const int Fb = in.F_base;

    for (int step = 0; step < in.T; ++step) {
        // ---- x_t of the 128 streams
        for (int e = tid; e < WG_STREAMS * F; e += WG_THREADS) {
            const int b = e / F, f = e - b * F;
            const long long i = base + b;
            float v = 0.f;
            if (i < n) {
                if (RING) {
                    const int fb = f < Fb ? f : f - Fb;
                    const float* row = ring_row(in, s_sid[b], s_rel[b], step);
                    const float cur = row ? row[fb] : 0.f;
                    if (f < Fb) v = cur;
                    else if (step > 0) {                   // add_deltas: delta[0] = 0
                        const float* prow = ring_row(in, s_sid[b], s_rel[b], step - 1);
                        v = cur - (prow ? prow[fb] : 0.f);
                    }
                } else {
                    v = input_value(in, i, step, f);
                }
            }
            A[b * AS + f] = v;
        }
        __syncthreads();
        // ---- phase 1: z and r of this warp's 16 units (n-tiles 2 w, 2 w + 1 of z and of r)
        if (active) {
#pragma unroll 1
            for (int mh = 0; mh < 2; ++mh) {
                float acc[4][4][4];
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int col = (q < 2 ? 0 : HP) + 16 * warp + 8 * (q & 1) + 2 * t;
                    const float b0 = __ldg(W.bias + col), b1 = __ldg(W.bias + col + 1);
#pragma unroll
                    for (int m = 0; m < 4; ++m) { acc[m][q][0] = b0; acc[m][q][1] = b1; acc[m][q][2] = b0; acc[m][q][3] = b1; }
                }
#pragma unroll 1
                for (int s = 0; s < KS; ++s) {
                    uint4 w[4];
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const int nt = (q < 2 ? 0 : NT2) + 2 * warp + (q & 1);
                        w[q] = __ldg(W.b1 + ((long long)s * NT1 + nt) * 32 + lane);
                    }
#pragma unroll
                    for (int m = 0; m < 4; ++m) {
                        uint32_t ah[4], al[4];
                        wg_afrag(A, AS, 16 * (4 * mh + m) + g, 8 * s + t, ah, al);
#pragma unroll
                        for (int q = 0; q < 4; ++q) {
                            mma_tf32(acc[m][q], al, w[q].x, w[q].y);
                            mma_tf32(acc[m][q], ah, w[q].z, w[q].w);
                            mma_tf32(acc[m][q], ah, w[q].x, w[q].y);
                        }
                    }
                }
#pragma unroll
                for (int m = 0; m < 4; ++m)
#pragma unroll
                    for (int q = 0; q < 4; ++q)
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const int row = 16 * (4 * mh + m) + g + 8 * (e >> 1), u = 16 * warp + 8 * (q & 1) + 2 * t + (e & 1);
                            const float gv = apply_ract(acc[m][q][e], W.ract);
                            if (q < 2) Z[row * RS + u] = gv;
                            else RH[row * RS + u] = gv * A[row * AS + FP + u];
                        }
            }
        }
        __syncthreads();
        // ---- phase 2: candidate from [x | r h], state update in place (no other warp reads h in this phase)
        if (active) {
#pragma unroll 1
            for (int mh = 0; mh < 2; ++mh) {
                float acc[4][2][4];
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    const int col = 2 * HP + 16 * warp + 8 * q + 2 * t;
                    const float b0 = __ldg(W.bias + col), b1 = __ldg(W.bias + col + 1);
#pragma unroll
                    for (int m = 0; m < 4; ++m) { acc[m][q][0] = b0; acc[m][q][1] = b1; acc[m][q][2] = b0; acc[m][q][3] = b1; }
                }
#pragma unroll 1
                for (int s = 0; s < KS; ++s) {
                    uint4 w[2];
#pragma unroll
                    for (int q = 0; q < 2; ++q) w[q] = __ldg(W.b2 + ((long long)s * NT2 + 2 * warp + q) * 32 + lane);
#pragma unroll
                    for (int m = 0; m < 4; ++m) {
                        uint32_t ah[4], al[4];
                        const int row = 16 * (4 * mh + m) + g;
                        if (s < KX) wg_afrag(A, AS, row, 8 * s + t, ah, al);
                        else wg_afrag(RH, RS, row, 8 * (s - KX) + t, ah, al);
#pragma unroll
                        for (int q = 0; q < 2; ++q) {
                            mma_tf32(acc[m][q], al, w[q].x, w[q].y);
                            mma_tf32(acc[m][q], ah, w[q].z, w[q].w);
                            mma_tf32(acc[m][q], ah, w[q].x, w[q].y);
                        }
                    }
                }
#pragma unroll
                for (int m = 0; m < 4; ++m)
#pragma unroll
                    for (int q = 0; q < 2; ++q)
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const int row = 16 * (4 * mh + m) + g + 8 * (e >> 1), u = 16 * warp + 8 * q + 2 * t + (e & 1);
                            const float zz = Z[row * RS + u], hp = A[row * AS + FP + u];
                            if constexpr (PIN_FMA) {
                                // gru_wide_kernel's SASS computes (q, e) = (0, 0) as fma(1 - z, a, z h) (it takes z h before
                                // the activation's branch) and every other (m, q, e) as fma(z, h, (1 - z) a), on both branches
                                const float a = apply_act(acc[m][q][e], W.act), om = __fsub_rn(1.f, zz);
                                A[row * AS + FP + u] = q == 0 && e == 0 ? __fmaf_rn(om, a, __fmul_rn(zz, hp))
                                                                        : __fmaf_rn(zz, hp, __fmul_rn(om, a));
                            } else {
                                A[row * AS + FP + u] = zz * hp + (1.f - zz) * apply_act(acc[m][q][e], W.act);
                            }
                        }
            }
        }
        __syncthreads();
    }
    // ---- Dense(1) + epilogue: warps 0..3 own the 128 streams
    if (tid < WG_STREAMS) {
        const long long i = base + tid;
        float logit = W.bd;
        for (int j = 0; j < H; ++j) logit = fmaf(A[tid * AS + FP + j], __ldg(W.wd + j), logit);
        epilogue(logit, i < n, i, s_sid[tid], dp, out);
    }
}

template <bool RING>
__global__ void __launch_bounds__(WG_THREADS, 1)
gru_wide_kernel(GruWideW W, K2In in, long long n, DecodeParams dp, K2Out out) {
    gru_wide_tile<RING, false>(W, in, [] { return (long long)blockIdx.x * WG_STREAMS; }, n, dp, out);
}

}  // namespace pb
