// gru_bank.cuh -- K2 for the fused family of networks (H <= 24, feature_size <= 16, no deltas, any activation pair): every
// such network of a model bank in ONE launch over the handle's shared MFCC ring, routed scans and the model pool.  One model
// alone (the default network's large-batch scan) runs the same arithmetic on warpgroup MMA in gru_wg.cuh.
//
// The per-step products run on the warp-level tensor cores in fp16 x 3 (hi / lo split of both operands, fp32 accumulate:
// a_lo b_hi + a_hi b_lo + a_hi b_hi) on mma.sync m16n8k16 / m16n8k8: one k16 + one k8 MMA per n-tile and pass cover the 24
// (padded) hidden units.  Pieces of 11 bits each, 22 bits per product like 3xTF32 (CPU emulation on the default network:
// 7.6e-8 vs 4.7e-8).  Hidden units sit in the k index in natural order (thread t of a quad holds units 8 tile + 2t, 2t + 1 in
// its accumulators = the (2t, 2t + 1) and (2t + 8, 2t + 9) k pairs of the A fragment), so h turns into the next step's A
// operand with two F2FP packs per n-tile and no data movement.
//
// A warp owns a 16-stream tile.  At each of the T steps it reads the tile's MFCC rows once, splits them into fp16 hi / lo A
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
// (x, y) -> half2 (x in the low half, as __floats2half2_rn), rounded to nearest and saturated to +-65504 instead of
// overflowing to +-inf.  PTX puts the first source operand in the upper half.  One F2FP.SATFINITE.F16.F32.PACK_AB.
__device__ __forceinline__ uint32_t pack_f16x2_sat(float x, float y) {
    uint32_t r;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(y), "f"(x));
    return r;
}
// (x, y) -> fp16 hi pair and the pair of residuals.  Exact fp16 x 3 operands for |v| < 65504; beyond that both pieces
// saturate, so the products see a finite operand of the same sign (|hi + lo| <= 131008) instead of inf - inf = NaN.
__device__ __forceinline__ void split_f16(float x, float y, uint32_t& hi, uint32_t& lo) {
    hi = pack_f16x2_sat(x, y);
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hi));
    lo = pack_f16x2_sat(x - f.x, y - f.y);
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

// Ring rows are staged per warp through shared memory, BANK_STAGE_STEPS steps at a time, two buffers: while the warp scans
// the steps of one buffer, 16-byte cp.async copies fill the other with the tile's rows of the next steps.  A lane pair owns one
// stream of the tile and copies its rows (32 B per lane pair and copy, 256 B per stream and buffer); zero rows (before a
// young stream's first frame, padding streams past n) are zero-filled by the copy itself (src-size 0).
constexpr int BANK_STAGE_STEPS = 4;
constexpr int BANK_STAGE_ROW = 16;                                   // floats per staged row: feature_size <= 16
constexpr int BANK_STAGE_BUF = BANK_STAGE_STEPS * 16 * BANK_STAGE_ROW;                   // floats: [step][stream][feature]
constexpr int BANK_STAGE_SMEM = (MMA_THREADS / 32) * 2 * BANK_STAGE_BUF * 4;             // 32 768 B per CTA
// Banks of up to two models stage; larger ones load ring rows directly, because the staging buffers would cost them a CTA
// per SM (shared memory: NM = 3, 4 drop from 3 CTAs to 2, NM = 6 .. 8 from 2 to 1) and that costs more than staging gains.
constexpr bool bank_stages(int nm, bool ring) { return ring && nm <= 2; }

__device__ __forceinline__ void cp_async16(float* dst, const float* src, uint32_t src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;"
                 :: "r"((uint32_t)__cvta_generic_to_shared(dst)), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int PENDING>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" :: "n"(PENDING) : "memory"); }

// This lane's share of steps t0 .. t0 + BANK_STAGE_STEPS - 1 of stream `cs` of the tile into buf: 16-byte pieces q = lane & 1 and
// 2 + (lane & 1) of each row.  cur is null-rowed for a padding stream (ok = false).
__device__ __forceinline__ void bank_stage(float* buf, const RingCursor& cur, bool ok, int cs, int t0, int T, const float* any, int lane) {
#pragma unroll
    for (int r = 0; r < BANK_STAGE_STEPS; ++r) {
        const float* row = ok && t0 + r < T ? cur.at(t0 + r) : nullptr;
        float* dst = buf + (r * 16 + cs) * BANK_STAGE_ROW;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int q = 2 * h + (lane & 1);
            const bool copy = row != nullptr && 4 * q < cur.stride;
            cp_async16(dst + 4 * q, copy ? row + 4 * q : any, copy ? 16u : 0u);
        }
    }
}

// The scan of one CTA: models m0 .. m0 + NM - 1 of P over the CTA's 64 entries, entries tile * 64 .. of n.  An entry is
// item e of the tick (stream in.ids[e], or e), or with a route list, list[e] = (item, stream).
// RING: rows from the stream ring (a tick), staged through shared memory up to NM = 2; otherwise from in.inputs,
// [n][T][F_base] contiguous (pb_predict), loaded directly.  KERAS_ACT: every model uses Keras's GRU defaults (recurrent hard_sigmoid, activation
// linear), compiled in; otherwise each model's pair is dispatched at run time.  Both compute the same expressions.
// PS: where P.w[k], P.dp[k] and P.o[k] come from (BankParams, or the model pool's per-model records, pool.cuh).
// WARP: the scan of one warp instead (NM = 1, RING): its 16 entries tile * 16 .., its model loaded by its own lanes into its
// own shared-memory slot (slot = warp), ring rows loaded directly.  The arithmetic is the same in every form.
template <int NM, bool RING, bool KERAS_ACT, class PS = BankParams, bool WARP = false>
__device__ __forceinline__ void bank_scan(const PS& P, int m0, const int2* list, long long tile, const K2In& in, long long n) {
    extern __shared__ __align__(16) unsigned char bank_smem[];
    static_assert(!WARP || (NM == 1 && RING), "a warp scans one model over the stream ring");
    const int ws = WARP ? (int)(threadIdx.x >> 5) : 0;                 // first shared-memory model slot of this scan
    const int l0 = WARP ? (int)(threadIdx.x & 31) : (int)threadIdx.x, ls = WARP ? 32 : (int)blockDim.x;
#pragma unroll 1
    for (int m = 0; m < NM; ++m) {
        const BankModelW& w = P.w[m0 + m];
        uint4* sf = reinterpret_cast<uint4*>(bank_smem + (ws + m) * BANK_MODEL_SMEM);
        float* sb = reinterpret_cast<float*>(sf + BANK_FRAG_U4);
        for (int e = l0; e < 2 * MMA_NT * 32; e += ls) sf[e] = __ldg(w.bfrag + e);
        for (int e = l0; e < MMA_NT * 32; e += ls) sf[2 * MMA_NT * 32 + e] = __ldg(w.xfrag + e);
        for (int e = l0; e < 72; e += ls) sb[e] = __ldg(w.bias + e);
        for (int e = l0; e < 24; e += ls) sb[72 + e] = __ldg(w.wd + e);
    }
    if (WARP) __syncwarp();
    else __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    const long long base = WARP ? tile * 16 : (tile * (MMA_THREADS / 32) + warp) * 16;
    if (base >= n) return;
    constexpr bool STAGE = bank_stages(NM, RING) && !WARP;
    const int F = in.F_base;
    long long idx[2];
    int sid[2];
    RingCursor rc[2];                                        // direct ring loads (RING && !STAGE)
    bool ok[2];
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
        idx[hf] = base + g + 8 * hf;
        ok[hf] = idx[hf] < n;
        sid[hf] = 0;
        if (list != nullptr && ok[hf]) {
            const int2 p = list[idx[hf]];
            idx[hf] = p.x;
            sid[hf] = p.y;
        } else if (RING && ok[hf]) {
            sid[hf] = in.ids ? in.ids[idx[hf]] : (int)idx[hf];
        }
        if (RING && ok[hf]) {
            if (!STAGE) {
                const long long ns = in.n_samples[sid[hf]];
                rc[hf].init(in, sid[hf], ns >= in.window ? (ns - in.window) / in.hop + 1 : 0);
            }
        }
    }
    // staging: this lane copies rows of stream cs = lane / 2 of the tile; chunk c of the window goes to buffer c & 1
    float* stage = reinterpret_cast<float*>(bank_smem + NM * BANK_MODEL_SMEM) + warp * 2 * BANK_STAGE_BUF;
    const int cs = lane >> 1;
    const bool cok = STAGE && base + cs < n;
    RingCursor cur;
    cur.stride = 0;
    if (cok) {
        const int csid = list != nullptr ? list[base + cs].y : in.ids ? in.ids[base + cs] : (int)(base + cs);
        const long long ns = in.n_samples[csid];
        cur.init(in, csid, ns >= in.window ? (ns - in.window) / in.hop + 1 : 0);
    }
    if (STAGE) {
        bank_stage(stage, cur, cok, cs, 0, in.T, in.ring, lane);
        cp_async_commit();
        bank_stage(stage + BANK_STAGE_BUF, cur, cok, cs, BANK_STAGE_STEPS, in.T, in.ring, lane);
        cp_async_commit();
    }
    int chunk = 0, cr = 0;                                   // step = chunk * BANK_STAGE_STEPS + cr
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
        if (STAGE) {
            if (cr == 0) {                                                  // chunk `chunk` has landed (the next may be in flight)
                cp_async_wait<1>();
                __syncwarp();
            }
            const float* xs = stage + (chunk & 1) * BANK_STAGE_BUF + cr * 16 * BANK_STAGE_ROW;
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
                const float* row = xs + (g + 8 * hf) * BANK_STAGE_ROW;
                const float2 lo = *reinterpret_cast<const float2*>(row + 2 * t), hi = *reinterpret_cast<const float2*>(row + 2 * t + 8);
                xv[hf][0] = 2 * t < F ? lo.x : 0.f;
                xv[hf][1] = 2 * t + 1 < F ? lo.y : 0.f;
                xv[hf][2] = 2 * t + 8 < F ? hi.x : 0.f;
                xv[hf][3] = 2 * t + 9 < F ? hi.y : 0.f;
            }
            if (cr + 1 == BANK_STAGE_STEPS) {                               // last step of the chunk: refill its buffer with chunk + 2
                __syncwarp();
                bank_stage(stage + (chunk & 1) * BANK_STAGE_BUF, cur, cok, cs, (chunk + 2) * BANK_STAGE_STEPS, in.T, in.ring, lane);
                cp_async_commit();
                cr = 0;
                ++chunk;
            } else {
                ++cr;
            }
        } else {
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
                const float* row = nullptr;                                 // stays nullptr: a row before the stream's first frame
                if (ok[hf]) row = RING ? rc[hf].next(step) : input_row(in, idx[hf], step);
                xv[hf][0] = (row != nullptr && 2 * t < F) ? __ldg(row + 2 * t) : 0.f;
                xv[hf][1] = (row != nullptr && 2 * t + 1 < F) ? __ldg(row + 2 * t + 1) : 0.f;
                xv[hf][2] = (row != nullptr && 2 * t + 8 < F) ? __ldg(row + 2 * t + 8) : 0.f;
                xv[hf][3] = (row != nullptr && 2 * t + 9 < F) ? __ldg(row + 2 * t + 9) : 0.f;
            }
        }
        uint32_t xh[4], xl[4];
        split_f16(xv[0][0], xv[0][1], xh[0], xl[0]);
        split_f16(xv[1][0], xv[1][1], xh[1], xl[1]);
        split_f16(xv[0][2], xv[0][3], xh[2], xl[2]);
        split_f16(xv[1][2], xv[1][3], xh[3], xl[3]);
#pragma unroll
        for (int m = 0; m < NM; ++m) {
            const uint4* sB = reinterpret_cast<const uint4*>(bank_smem + (ws + m) * BANK_MODEL_SMEM);
            const uint4* sX = sB + 2 * MMA_NT * 32;
            const float* sBias = reinterpret_cast<const float*>(sB + BANK_FRAG_U4);
            const int ra = P.w[m0 + m].ract, ac = P.w[m0 + m].act;
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
                    for (int e = 0; e < 4; ++e) {
                        const float r = KERAS_ACT ? hard_sigmoid(acc[3 + nt][e]) : apply_ract(acc[3 + nt][e], ra);
                        rh[nt][e] = __fmul_rn(r, hreg[m][nt][e]);
                    }
                uint32_t ah[4], al[4], ch[2], cl[2];
                frag_f16(rh, ah, al, ch, cl);
                mma3_f16(acc, 6, ah, al, ch, cl, sB, lane);
            }
            // h = z h + (1 - z) a, rounded as fma(z, h, (1 - z) a) in every specialisation
#pragma unroll
            for (int nt = 0; nt < 3; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float z = KERAS_ACT ? hard_sigmoid(acc[nt][e]) : apply_ract(acc[nt][e], ra);
                    const float a = KERAS_ACT ? acc[6 + nt][e] : apply_act(acc[6 + nt][e], ac);
                    hreg[m][nt][e] = __fmaf_rn(z, hreg[m][nt][e], __fmul_rn(__fsub_rn(1.f, z), a));
                }
        }
    }
    if (STAGE) cp_async_wait<0>();                                    // copies of chunks past the window
    // ---- per model: Dense(1) (per-thread partial over its 6 units per row, reduced over the quad) and the epilogue
#pragma unroll
    for (int m = 0; m < NM; ++m) {
        const float* sWd = reinterpret_cast<const float*>(bank_smem + (ws + m) * BANK_MODEL_SMEM + BANK_FRAG_U4 * 16) + 72;
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
            epilogue(part + P.w[m0 + m].bd, t == 0 && ok[hf], idx[hf], sid[hf], P.dp[m0 + m], P.o[m0 + m]);
        }
    }
}

// Every model of P over the n items of a tick (or of pb_predict's inputs), 64 items per CTA.
template <int NM, bool RING, bool KERAS_ACT>
__global__ void __launch_bounds__(MMA_THREADS, 1)                    // NM >= 2: one model runs in gru_wg_kernel (gru_wg.cuh)
gru_bank_kernel(const __grid_constant__ BankParams P, K2In in, long long n) {
    bank_scan<NM, RING, KERAS_ACT>(P, 0, nullptr, blockIdx.x, in, n);
}

// Per-stream model subscriptions: route_kernel has listed, for each model m, the (item, stream) pairs of the tick whose
// stream subscribes to m (count[m] of them).  A routed launch scans models 0 .. nm - 1 of P; model k takes CTAs
// tile0[k] .. tile0[k + 1] - 1, 64 list entries each, sized on the host from the model's subscriber count.
struct BankRoute {
    const int2* list[BANK_MAX_MODELS];           // model k's list
    const unsigned* count[BANK_MAX_MODELS];      // ... and its length (device)
    int tile0[BANK_MAX_MODELS + 1];
    int nm;
};

// Outputs and lists of route_kernel.  Outputs are model-major [M][n] (M = 1: pb_update's [n]); raw and fired may be null.
struct RouteOut {
    float* raw;
    double* conf;
    uint8_t* fired;
    int M;
    int2* lists;                     // [BANK_MAX_MODELS][list_stride] (item, stream) pairs, or null: NaN fill only
    long long list_stride;
    unsigned* count;                 // [BANK_MAX_MODELS] list lengths, zeroed before the launch
    unsigned listed;                 // bit m: model m is scanned from its list
};

// One thread per tick item.  For every model m < M whose bit the item's stream lacks: raw = conf = NaN, fired = 0 (the only
// place that writes them).  For every listed model whose bit it has: appends (item, stream) to m's list, one atomicAdd per
// warp and model.  The order within a list varies; a window's score does not depend on its tile.
__global__ void __launch_bounds__(256) route_kernel(const uint8_t* route, const int* ids, long long n, RouteOut r) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool ok = i < n;
    const int sid = ok ? (ids ? ids[i] : (int)i) : 0;
    const unsigned mask = ok ? route[sid] : 0u;
    const int lane = threadIdx.x & 31;
    for (int m = 0; m < r.M; ++m) {
        const unsigned bit = 1u << m;
        const long long o = (long long)m * n + i;
        if (ok && !(mask & bit)) {
            if (r.raw) r.raw[o] = __int_as_float(0x7fc00000);
            r.conf[o] = __longlong_as_double(0x7ff8000000000000LL);
            if (r.fired) r.fired[o] = 0;
        }
        if (r.lists != nullptr && (r.listed & bit)) {                 // uniform over the grid
            const bool sub = ok && (mask & bit);
            const unsigned b = __ballot_sync(0xffffffffu, sub);
            if (b == 0) continue;
            unsigned at = 0;
            if (lane == 0) at = atomicAdd(r.count + m, (unsigned)__popc(b));
            at = __shfl_sync(0xffffffffu, at, 0);
            if (sub) r.lists[m * r.list_stride + at + __popc(b & ((1u << lane) - 1u))] = make_int2((int)i, sid);
        }
    }
}

// One model per CTA (NM = 1, with its staging and, for KERAS_ACT, the compiled-in activations); a CTA past its model's
// list exits before it loads any weights.  Outputs go to item list[e].x, the trigger update to stream list[e].y; per model
// the accumulation order is the bank's, so a pair scores bit-identically routed and unrouted.
template <bool KERAS_ACT>
__global__ void __launch_bounds__(MMA_THREADS, 4)
gru_bank_routed_kernel(const __grid_constant__ BankParams P, const __grid_constant__ BankRoute R, K2In in) {
    int k = 0;
    while (k + 1 < R.nm && (int)blockIdx.x >= R.tile0[k + 1]) ++k;
    const long long tile = (long long)blockIdx.x - R.tile0[k];
    const long long n = *R.count[k];
    if (tile * (MMA_THREADS / 32) * 16 >= n) return;
    bank_scan<1, true, KERAS_ACT>(P, k, R.list[k], tile, in, n);
}

}  // namespace pb
