// train_wide.cuh -- training of networks up to 128 GRU units (pb_train_wide, pb_train_wide_loss) on the tensor cores.  Same
// contract and arithmetic as train.cuh (GRU with reset_after = False, Dense(1, sigmoid), the
// weighted log loss, per-gate input dropout, RMSprop), with rows of TW_STRIDE floats.  Every matrix product runs on
// mma.sync.m16n8k8 TF32 as 3xTF32 (al bh + ah bl + ah bh, fp32 accumulators), with both halves rounded to nearest (tw_split)
// rather than gru_wide.cuh's truncating split_tf32: truncation leaves up to 2^-20 of each product, about 20 times float32's
// error on a single product, which fails the training tests' bound of 10 times float32's (DESIGN section 6); rounding leaves
// about 2^-22.  Accumulation across k-steps is in fp32 registers (tw_mma).  The elementwise work is float32 as in
// train.cuh, with hard_sigmoid's argument rounded by tr_hard_sigmoid_arg.
// The Dense layer's dot products (one output column) and the dense gradient run on the CUDA cores in float32.
//
//   train_wide_scan_kernel  one CTA of 4 warps per (tile of TR_TILE entries, 16 of its entries): the 16 entries are one m16
//                           row block.  Forward, per step: the masked inputs x m_g of the three gates are staged in shared
//                           memory, then [x m_z | h] [K_z; U_z] and [x m_r | h] [K_r; U_r] (warps over the n-tiles of 8
//                           units), then [x m_h | r h] [K_h; U_h].  The weight fragments come from L2 each step, as
//                           gru_wide_kernel takes them (a row is 223 KB: its hi / lo pairs would not fit shared memory), and
//                           are split on the fly because RMSprop changes them every batch.  Each (entry, step) record of the
//                           tile's state keeps x m_g, h, r h and the pre-activations.  Backward runs the dh chain over the
//                           steps: dah U_h^T, then [daz | dar] [U_z^T; U_r^T] on the tensor cores, and overwrites the
//                           pre-activations with the gate gradients.
//   train_wide_grad_kernel  one CTA per (tile, 16 rows of the gradient, gate): the gradient of kernel, recurrent and bias is one
//                           (F + H + 1) x 3H matrix in the row layout, A^T D over K = the tile's entries x steps, A the
//                           records' [x m_g | h or r h | 1] and D the gate gradients; the column of ones makes the bias
//                           gradient (the column sums) a product too.  K runs step by step, 8 entries at a time, so the sum
//                           order is fixed.  The (tile, 0, z) CTA adds dense_w's and dense_b's gradients and the tile's
//                           loss sum in entry order.
// The tiles' partial rows are summed in tile order by train_update_kernel<TW_STRIDE> (train.cuh), which applies RMSprop or
// writes the gradient; shuffle keys and the segmented sort are train.cuh's.  No float atomics anywhere: a tile's partial row
// depends only on its own entries, so results are independent of the other rows, of the workspace grouping and of how
// the tiles of a batch are cut into launches.
//
// State: a tile's state is tw_tile_floats(T, F, H) floats, T TR_TILE records of tw_rec(F, H) = 3 FP + 5 HP floats (FP, HP:
// F and H rounded up to 8) plus a per-entry tail, so about 4 T (3 FP + 5 HP) bytes per entry: 308 KB at T = 112, F = 16,
// H = 128, 43 KB at the default front end (T 29, F 13) and H = 64.  The tiles of a batch run in launches whose state stays
// under TW_STATE_CAP; a partial row is TW_STRIDE floats (223 KB) per tile of the batch.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "gru_kernels.cuh"
#include "train.cuh"

namespace pb {

constexpr int TW_STRIDE = 55812;           // floats per weight row: 3 H (F + H + 1) + H + 1 <= 55 809 (H = 128, F = 16)
constexpr int TW_MAX_H = 128;
constexpr int TW_SUB = 16;                 // entries per scan CTA (one m16 row block)
constexpr int TW_THREADS = 128;
constexpr int TW_XS = 16 + 4;              // shared row strides (4 mod 32 words: conflict-free A fragment loads)
constexpr int TW_HS = TW_MAX_H + 4;
constexpr int TW_MBLOCKS = (TR_MAX_F + TW_MAX_H + 1 + 15) / 16;   // 16-row blocks of the (F + H + 1) x 3H gradient
constexpr size_t TW_STATE_CAP = size_t(512) << 20;                 // state of one launch's tiles

__host__ __device__ constexpr int tw_fp(int F) { return (F + 7) & ~7; }
__host__ __device__ constexpr int tw_hp(int H) { return (H + 7) & ~7; }
// One (entry, step) record: x m_z, x m_r, x m_h [FP each], then h (the step's starting state), r h, az | daz, ar | dar,
// ah | dah [HP each].
__host__ __device__ constexpr int tw_rec(int F, int H) { return 3 * tw_fp(F) + 5 * tw_hp(H); }
// A tile's state: records [T][TR_TILE], then per entry its loss (double), dlogit, and h_T [HP]; 256-byte aligned.
__host__ __device__ constexpr long long tw_tile_floats(int T, int F, int H) {
    return ((long long)T * TR_TILE * tw_rec(F, H) + TR_TILE * (3 + tw_hp(H)) + 63) / 64 * 64;
}

struct TrainWideScan {
    const float* weights;            // [k][TW_STRIDE]
    const TrainRowDev* rows;
    const float* inputs;             // [n_rec][T][F]
    const uint8_t* targets;
    const int* ent;                  // group-local entry -> clip
    const int* order;                // group-local visiting order, or null
    const TrainTile* tiles;          // this launch's tiles
    const long long* soff;           // [tiles] each tile's state offset (floats) in `state`
    float* state;
    int T, F;
    long long epoch;
    float rate, scale, loss_bias;
};

struct TrainWideGrad {
    const TrainRowDev* rows;
    const TrainTile* tiles;
    const long long* soff;
    const float* state;
    float* part;                     // [tiles of the batch][TW_STRIDE]
    double* part_loss;
    int p0;                          // the batch's index of this launch's first tile
    int T, F;
};

// v = hi + lo + O(2^-22 v), hi and lo TF32 rounded to nearest (cvt.rna; v - hi is exact in fp32).
__device__ __forceinline__ void tw_split(float v, uint32_t& hi, uint32_t& lo) {
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hi) : "f"(v));
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lo) : "f"(v - __uint_as_float(hi)));
}

// acc += A[16][K] B[K][8] on the tensor cores with the 3xTF32 split: A fp32 in shared memory (row stride as, K a multiple
// of 8), bk(k) the lane's B element (row k, column g), 0 outside the matrix.  Each k-step's three products go to a zeroed
// fragment that is added to acc with IEEE float adds: the tensor cores' own fp32 accumulation truncates, and over the K of
// the weight-gradient products (entries x steps, up to 7 168) that bias grows linearly.
template <class BK>
__device__ __forceinline__ void tw_mma(float (&acc)[4], const float* A, int as, int K, BK bk) {
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
#pragma unroll 2
    for (int k = 0; k < K; k += 8) {
        const float v[4] = {A[g * as + k + t], A[(g + 8) * as + k + t], A[g * as + k + t + 4], A[(g + 8) * as + k + t + 4]};
        uint32_t ah[4], al[4], bh0, bh1, bl0, bl1;
#pragma unroll
        for (int e = 0; e < 4; ++e) tw_split(v[e], ah[e], al[e]);
        tw_split(bk(k + t), bh0, bl0);
        tw_split(bk(k + t + 4), bh1, bl1);
        float d[4] = {0.f, 0.f, 0.f, 0.f};
        mma_tf32(d, al, bh0, bh1);
        mma_tf32(d, ah, bl0, bl1);
        mma_tf32(d, ah, bh0, bh1);
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[e] += d[e];
    }
}

__global__ void __launch_bounds__(TW_THREADS) train_wide_scan_kernel(const __grid_constant__ TrainWideScan S) {
    __shared__ __align__(16) float xs[3][TW_SUB][TW_XS];      // the step's x m_g
    __shared__ __align__(16) float hs[TW_SUB][TW_HS];         // h; backward: dh (then dh z + drh r, then dh_(t-1))
    __shared__ __align__(16) float zs[TW_SUB][TW_HS];         // z; backward: daz
    __shared__ __align__(16) float rhs[TW_SUB][TW_HS];        // r h; backward: dah
    __shared__ __align__(16) float b4[TW_SUB][TW_HS];         // backward: dar
    __shared__ float mk[TW_SUB][3 * TR_MAX_F];                 // mask value of (entry, 3 f + g): scale or 0
    __shared__ int s_rec[TW_SUB], s_jj[TW_SUB];
    __shared__ float s_dl[TW_SUB];
    const TrainTile tile = S.tiles[blockIdx.x];
    const int e0 = blockIdx.y * TW_SUB;
    if (e0 >= tile.count) return;
    const TrainRowDev rd = S.rows[tile.row];
    const int H = rd.hidden, F = S.F, T = S.T, H3 = 3 * H, FP = tw_fp(F), HP = tw_hp(H), R = tw_rec(F, H), NT = HP / 8;
    const int OH = 3 * FP, ORH = OH + HP, OZ = ORH + HP, OR = OZ + HP, OA = OR + HP;
    const float* K = S.weights + (size_t)tile.row * TW_STRIDE;
    const float* U = K + F * H3;
    const float* bias = U + H * H3;
    const float* dw = bias + H3;
    const float db = dw[H];
    float* st = S.state + S.soff[blockIdx.x];
    auto rec = [&](int t, int e) { return st + ((size_t)t * TR_TILE + e0 + e) * R; };
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t4 = lane & 3;
    for (int i = tid; i < 3 * TW_SUB * TW_XS; i += TW_THREADS) (&xs[0][0][0])[i] = 0.f;
    for (int i = tid; i < TW_SUB * TW_HS; i += TW_THREADS) {
        (&hs[0][0])[i] = 0.f; (&zs[0][0])[i] = 0.f; (&rhs[0][0])[i] = 0.f; (&b4[0][0])[i] = 0.f;
    }
    if (tid < TW_SUB) {
        const int i = e0 + tid;
        int jj = -1, r = -1;
        if (i < tile.count) {
            const int pos = tile.start + i;
            jj = S.order ? S.order[tile.base + pos] : pos;
            r = S.ent[tile.base + jj];
        }
        s_jj[tid] = jj; s_rec[tid] = r;
    }
    __syncthreads();
    for (int i = tid; i < TW_SUB * 3 * F; i += TW_THREADS) {
        const int e = i / (3 * F), c = i - e * 3 * F;
        float m = 0.f;
        if (s_jj[e] >= 0) {
            m = S.scale;
            if (S.rate > 0.f) {
                const uint64_t base = tr_entry(rd.seed, (uint64_t)S.epoch, (uint64_t)s_jj[e]);
                const float u = (float)(unsigned)(tr_mix(base + 1 + c) >> 40) * 5.9604644775390625e-8f;
                if (!(u >= S.rate)) m = 0.f;
            }
        }
        mk[e][c] = m;
    }
    __syncthreads();

    // ---- forward
#pragma unroll 1
    for (int t = 0; t < T; ++t) {
        for (int i = tid; i < TW_SUB * F; i += TW_THREADS) {
            const int e = i / F, f = i - e * F;
            const float x = s_rec[e] >= 0 ? __ldg(S.inputs + ((size_t)s_rec[e] * T + t) * F + f) : 0.f;
            float* rc = rec(t, e);
#pragma unroll
            for (int q = 0; q < 3; ++q) {
                const float v = x * mk[e][3 * f + q];
                xs[q][e][f] = v;
                rc[q * FP + f] = v;
            }
        }
        for (int i = tid; i < TW_SUB * H; i += TW_THREADS) {
            const int e = i / H, u = i - e * H;
            rec(t, e)[OH + u] = hs[e][u];
        }
        __syncthreads();
        // z and r: n-tiles [0, NT) of z, [NT, 2 NT) of r
#pragma unroll 1
        for (int q = warp; q < 2 * NT; q += TW_THREADS / 32) {
            const int gate = q < NT ? 0 : 1, n0 = 8 * (q - gate * NT), u = n0 + g, col = gate * H + u;
            const bool ok = u < H;
            float acc[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) { const int c = n0 + 2 * t4 + (e & 1); acc[e] = c < H ? bias[gate * H + c] : 0.f; }
            tw_mma(acc, &xs[gate][0][0], TW_XS, FP, [&](int k) { return ok && k < F ? __ldg(K + (size_t)k * H3 + col) : 0.f; });
            tw_mma(acc, &hs[0][0], TW_HS, HP, [&](int k) { return ok && k < H ? __ldg(U + (size_t)k * H3 + col) : 0.f; });
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int row = g + 8 * (e >> 1), c = n0 + 2 * t4 + (e & 1);
                if (c >= H) continue;
                float* rc = rec(t, row);
                const float v = tr_ract(rd.ract, acc[e]);
                if (gate == 0) {
                    rc[OZ + c] = acc[e];
                    zs[row][c] = v;
                } else {
                    rc[OR + c] = acc[e];
                    const float rh = v * hs[row][c];
                    rhs[row][c] = rh;
                    rc[ORH + c] = rh;
                }
            }
        }
        __syncthreads();
        // candidate and the new h (no warp reads h in this phase)
#pragma unroll 1
        for (int q = warp; q < NT; q += TW_THREADS / 32) {
            const int n0 = 8 * q, u = n0 + g, col = 2 * H + u;
            const bool ok = u < H;
            float acc[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) { const int c = n0 + 2 * t4 + (e & 1); acc[e] = c < H ? bias[2 * H + c] : 0.f; }
            tw_mma(acc, &xs[2][0][0], TW_XS, FP, [&](int k) { return ok && k < F ? __ldg(K + (size_t)k * H3 + col) : 0.f; });
            tw_mma(acc, &rhs[0][0], TW_HS, HP, [&](int k) { return ok && k < H ? __ldg(U + (size_t)k * H3 + col) : 0.f; });
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int row = g + 8 * (e >> 1), c = n0 + 2 * t4 + (e & 1);
                if (c >= H) continue;
                rec(t, row)[OA + c] = acc[e];
                const float hh = tr_act(rd.act, acc[e]), z = zs[row][c];
                hs[row][c] = fmaf(z, hs[row][c], (1.f - z) * hh);
            }
        }
        __syncthreads();
    }

    // ---- Dense + sigmoid + loss (train.cuh's formulas); entries past the tile's count have dlogit 0
    double* tl_loss = reinterpret_cast<double*>(st + (size_t)T * TR_TILE * R);
    float* tl_dl = reinterpret_cast<float*>(tl_loss + TR_TILE);
    float* tl_h = tl_dl + TR_TILE;
    if (tid < TW_SUB) {
        float lg = 0.f;
        for (int j = 0; j < H; ++j) lg = fmaf(hs[tid][j], dw[j], lg);
        const float logit = lg + db;
        const float p = 1.f / (1.f + expf(-logit));
        double loss = 0.0;
        float dlogit = 0.f;
        if (s_rec[tid] >= 0) {
            const float y = S.targets[s_rec[tid]] ? 1.f : 0.f, lb = S.loss_bias;
            loss = (double)(lb * (-(1.f - y) * logf(1.f - p + 1e-7f)) + (1.f - lb) * (-y * logf(p + 1e-7f)));
            const float dp = (lb * (1.f - y) / (1.f - p + 1e-7f) - (1.f - lb) * y / (p + 1e-7f)) * (1.f / (float)tile.batch);
            dlogit = dp * (p * (1.f - p));
        }
        tl_loss[e0 + tid] = loss;
        tl_dl[e0 + tid] = dlogit;
        s_dl[tid] = dlogit;
    }
    __syncthreads();
    for (int i = tid; i < TW_SUB * H; i += TW_THREADS) {
        const int e = i / H, j = i - e * H;
        tl_h[(size_t)(e0 + e) * HP + j] = hs[e][j];
        hs[e][j] = s_dl[e] * dw[j];
    }
    __syncthreads();

    // ---- BPTT
#pragma unroll 1
    for (int t = T - 1; t >= 0; --t) {
        for (int i = tid; i < TW_SUB * H; i += TW_THREADS) {
            const int e = i / H, j = i - e * H;
            float* rc = rec(t, e);
            const float az = rc[OZ + j], ah = rc[OA + j], hp = rc[OH + j], dh = hs[e][j];
            const float z = tr_ract(rd.ract, az), hh = tr_act(rd.act, ah);
            const float daz = dh * (hp - hh) * tr_ract_grad(rd.ract, az, z);
            const float dah = dh * (1.f - z) * tr_act_grad(rd.act, hh);
            rc[OZ + j] = daz; rc[OA + j] = dah;
            zs[e][j] = daz; rhs[e][j] = dah;
            hs[e][j] = dh * z;
        }
        __syncthreads();
        // drh = dah U_h^T (B[k = c][n = q] = U[q][2H + c]); dar; dh z + drh r
#pragma unroll 1
        for (int q = warp; q < NT; q += TW_THREADS / 32) {
            const int n0 = 8 * q, u = n0 + g;
            const bool ok = u < H;
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
            tw_mma(acc, &rhs[0][0], TW_HS, HP, [&](int k) { return ok && k < H ? __ldg(U + (size_t)u * H3 + 2 * H + k) : 0.f; });
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int row = g + 8 * (e >> 1), c = n0 + 2 * t4 + (e & 1);
                if (c >= H) continue;
                float* rc = rec(t, row);
                const float ar = rc[OR + c], hp = rc[OH + c];
                const float r = tr_ract(rd.ract, ar);
                const float dar = acc[e] * hp * tr_ract_grad(rd.ract, ar, r);
                rc[OR + c] = dar;
                b4[row][c] = dar;
                hs[row][c] = fmaf(acc[e], r, hs[row][c]);
            }
        }
        __syncthreads();
        // dh_(t-1) = (dh z + drh r) + daz U_z^T + dar U_r^T
#pragma unroll 1
        for (int q = warp; q < NT; q += TW_THREADS / 32) {
            const int n0 = 8 * q, u = n0 + g;
            const bool ok = u < H;
            float acc[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) { const int c = n0 + 2 * t4 + (e & 1); acc[e] = c < H ? hs[g + 8 * (e >> 1)][c] : 0.f; }
            tw_mma(acc, &zs[0][0], TW_HS, HP, [&](int k) { return ok && k < H ? __ldg(U + (size_t)u * H3 + k) : 0.f; });
            tw_mma(acc, &b4[0][0], TW_HS, HP, [&](int k) { return ok && k < H ? __ldg(U + (size_t)u * H3 + H + k) : 0.f; });
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int row = g + 8 * (e >> 1), c = n0 + 2 * t4 + (e & 1);
                if (c < H) hs[row][c] = acc[e];
            }
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(TW_THREADS) train_wide_grad_kernel(const __grid_constant__ TrainWideGrad P) {
    const TrainTile tile = P.tiles[blockIdx.x];
    const int H = P.rows[tile.row].hidden, F = P.F, T = P.T, H3 = 3 * H, FP = tw_fp(F), HP = tw_hp(H), R = tw_rec(F, H);
    const int M = F + H + 1, gate = blockIdx.z, m0 = 16 * blockIdx.y;
    if (m0 >= M) return;
    const int OH = 3 * FP, ORH = OH + HP, OD = ORH + HP + gate * HP;     // OD: this gate's gradient slot
    const float* st = P.state + P.soff[blockIdx.x];
    float* out = P.part + (size_t)(P.p0 + blockIdx.x) * TW_STRIDE;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t4 = lane & 3;
    // the lane's two A rows: a record offset, -1 for the row of ones, -2 past the matrix
    auto src = [&](int m) { return m < F ? gate * FP + m : m < F + H ? (gate == 2 ? ORH : OH) + (m - F) : m == F + H ? -1 : -2; };
    const int s0 = src(m0 + g), s1 = src(m0 + g + 8);
    auto av = [](const float* rc, int s) { return s >= 0 ? rc[s] : s == -1 ? 1.f : 0.f; };
    const int NT = HP / 8;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[i][e] = 0.f;
    const int KE = (tile.count + 7) & ~7;
#pragma unroll 1
    for (int t = 0; t < T; ++t) {
#pragma unroll 1
        for (int kb = 0; kb < KE; kb += 8) {
            const float* r0 = st + ((size_t)t * TR_TILE + kb + t4) * R;     // records k and k + 4 of this lane
            const float* r1 = r0 + 4 * (size_t)R;
            const float v[4] = {av(r0, s0), av(r0, s1), av(r1, s0), av(r1, s1)};
            uint32_t ah[4], al[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) tw_split(v[e], ah[e], al[e]);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int u = 8 * (warp + 4 * i) + g;
                if (warp + 4 * i >= NT) continue;
                uint32_t bh0, bh1, bl0, bl1;
                tw_split(u < H ? r0[OD + u] : 0.f, bh0, bl0);
                tw_split(u < H ? r1[OD + u] : 0.f, bh1, bl1);
                float d[4] = {0.f, 0.f, 0.f, 0.f};
                mma_tf32(d, al, bh0, bh1);
                mma_tf32(d, ah, bl0, bl1);
                mma_tf32(d, ah, bh0, bh1);
#pragma unroll
                for (int e = 0; e < 4; ++e) acc[i][e] += d[e];
            }
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        if (warp + 4 * i >= NT) continue;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int m = m0 + g + 8 * (e >> 1), c = 8 * (warp + 4 * i) + 2 * t4 + (e & 1);
            if (m < M && c < H) out[(size_t)m * H3 + gate * H + c] = acc[i][e];
        }
    }
    if (blockIdx.y == 0 && gate == 0) {
        const double* tl_loss = reinterpret_cast<const double*>(st + (size_t)T * TR_TILE * R);
        const float* tl_dl = reinterpret_cast<const float*>(tl_loss + TR_TILE);
        const float* tl_h = tl_dl + TR_TILE;
        for (int j = tid; j <= H; j += TW_THREADS) {
            float a = 0.f;
            for (int e = 0; e < tile.count; ++e) a = j < H ? fmaf(tl_h[(size_t)e * HP + j], tl_dl[e], a) : a + tl_dl[e];
            out[(size_t)M * H3 + j] = a;
        }
        if (tid == 0) {
            double a = 0.0;
            for (int e = 0; e < tile.count; ++e) a += tl_loss[e];
            P.part_loss[P.p0 + blockIdx.x] = a;
        }
    }
}

}  // namespace pb
