// gru_wg.cuh -- K2 of the default network and of every one-model fused-family launch (launch_bank_act with NM = 1) on
// warpgroup MMA (wgmma.mma_async, sm_90a) instead of per-warp mma.sync.
//
// A = 64 x 16 fp16 from registers: warp w of the warpgroup holds rows 16 w .. 16 w + 15 in the layout of mma.m16n8k16's A
// fragment.  B = 16 x N fp16 in shared memory, K-major without swizzle: 8 x 8 core matrices of 128 contiguous bytes, element
// (k, n) at byte (n / 8) * 256 + (k / 8) * 128 + (n % 8) * 16 + (k % 8) * 2 of its tile (LBO 128, SBO 256).  D = 64 x N f32 in
// registers, n8 block j in d[4 j .. 4 j + 3] laid out as mma.m16n8's C fragment.  So h stays in accumulator layout and
// becomes the next step's A operand as in bank_scan, and units 16..23 run as a k16 whose upper 8 k-slots are zero in A and B.
// Per accumulator the products come in bank_scan's order (bias, x part, h part, pass by pass, k16 before k8); wgmma adds
// them bit-identically to mma.sync (scripts/wgmma_probe.cu, DESIGN.md §6 "wgmma probe"), so both scans give the same bits.
#pragma once
#include <stdint.h>

#include "gru_bank.cuh"

namespace pb {

constexpr int WG_TILE_BYTES = 72 * 16 * 2;               // one k16 x n72 fp16 B tile
// byte offset of element (k, n) of a B tile
__host__ __device__ constexpr int wg_b_offset(int k, int n) { return (n >> 3) * 256 + (k >> 3) * 128 + (n & 7) * 16 + (k & 7) * 2; }

// Matrix descriptor of the B tile at p (shared memory, 16-byte aligned): start address, LBO = 128, SBO = 256, no swizzle.
__device__ __forceinline__ uint64_t wg_desc(const void* p) {
    const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
    return (uint64_t)((a & 0x3ffff) >> 4) | ((uint64_t)(128 >> 4) << 16) | ((uint64_t)(256 >> 4) << 32);
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" :: "n"(N) : "memory"); }
// Generic-proxy writes of B tiles become visible to wgmma (async proxy) reads; then a CTA barrier.
__device__ __forceinline__ void wg_fence_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// Keeps the compiler from moving reads of accumulator registers above the wgmma.wait_group that completes them.
template <int N>
__device__ __forceinline__ void wg_fence_regs(float* d) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i]) :: "memory");
}

// d[0 .. N / 2) += A . B, A from registers (a), B from shared memory (desc)
__device__ __forceinline__ void wgmma_n24(float* d, const uint32_t (&a)[4], uint64_t desc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %17, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n24k16.f32.f16.f16 "
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, %16, p, 1, 1, 0;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(1));
}
__device__ __forceinline__ void wgmma_n48(float* d, const uint32_t (&a)[4], uint64_t desc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %29, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 "
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}, "
                 "{%24,%25,%26,%27}, %28, p, 1, 1, 0;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(1));
}
__device__ __forceinline__ void wgmma_n72(float* d, const uint32_t (&a)[4], uint64_t desc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %41, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n72k16.f32.f16.f16 "
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,"
                 "%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35}, {%36,%37,%38,%39}, %40, p, 1, 1, 0;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
                   "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(1));
}

// The one-model scan of a CTA = one warpgroup over entries tile * 64 .. of n, with bank_scan<1, RING, KERAS_ACT>'s inputs,
// staging and epilogue.  The weights are staged once per CTA: the fragments upload_frag16 built are scattered into six B
// tiles (input weights hi / lo, recurrent units 0..15 hi / lo, units 16..23 hi / lo).  wgmma is warpgroup-collective, so every
// warp runs all T steps; entries past n are padding (zero rows, no output).
template <bool RING, bool KERAS_ACT>
__global__ void __launch_bounds__(MMA_THREADS, 4)
gru_wg_kernel(const __grid_constant__ BankParams P, K2In in, long long n) {
    extern __shared__ __align__(16) unsigned char bank_smem[];
    const BankModelW& w = P.w[0];
    unsigned char* sW = bank_smem;                                              // 6 tiles of WG_TILE_BYTES
    float* sb = reinterpret_cast<float*>(bank_smem + BANK_FRAG_U4 * 16);       // bias [72], dense weights [24]
    for (int e = threadIdx.x; e < 3 * MMA_NT * 32; e += blockDim.x) {
        // e = (kt * MMA_NT + nt) * 32 + lane, kt 0, 1 recurrent, 2 input; (x, y, z, w) = hi k 2t, hi k 2t + 8, lo k 2t, lo k 2t + 8
        const int kt = e / (MMA_NT * 32), nt = (e / 32) % MMA_NT, lane = e & 31, col = 8 * nt + (lane >> 2), k = 2 * (lane & 3);
        const uint4 f = kt < 2 ? __ldg(w.bfrag + e) : __ldg(w.xfrag + e - 2 * MMA_NT * 32);
        unsigned char* hi = sW + (kt == 2 ? 0 : 2 + 2 * kt) * WG_TILE_BYTES;
        unsigned char* lo = hi + WG_TILE_BYTES;
        *reinterpret_cast<uint32_t*>(hi + wg_b_offset(k, col)) = f.x;
        *reinterpret_cast<uint32_t*>(hi + wg_b_offset(k + 8, col)) = f.y;
        *reinterpret_cast<uint32_t*>(lo + wg_b_offset(k, col)) = f.z;
        *reinterpret_cast<uint32_t*>(lo + wg_b_offset(k + 8, col)) = f.w;
    }
    for (int e = threadIdx.x; e < 72; e += blockDim.x) sb[e] = __ldg(w.bias + e);
    for (int e = threadIdx.x; e < 24; e += blockDim.x) sb[72 + e] = __ldg(w.wd + e);
    wg_fence_smem();
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    const long long base = ((long long)blockIdx.x * (MMA_THREADS / 32) + warp) * 16;
    constexpr bool STAGE = RING;
    const int F = in.F_base;
    long long idx[2];
    int sid[2];
    bool ok[2];
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
        idx[hf] = base + g + 8 * hf;
        ok[hf] = idx[hf] < n;
        sid[hf] = RING && ok[hf] ? (in.ids ? in.ids[idx[hf]] : (int)idx[hf]) : 0;
    }
    float* stage = reinterpret_cast<float*>(bank_smem + BANK_MODEL_SMEM) + warp * 2 * BANK_STAGE_BUF;
    const int cs = lane >> 1;
    const bool cok = STAGE && base + cs < n;
    RingCursor cur;
    cur.stride = 0;
    if (cok) {
        const int csid = in.ids ? in.ids[base + cs] : (int)(base + cs);
        const long long ns = in.n_samples[csid];
        cur.init(in, csid, ns >= in.window ? (ns - in.window) / in.hop + 1 : 0);
    }
    if (STAGE) {
        bank_stage(stage, cur, cok, cs, 0, in.T, in.ring, lane);
        cp_async_commit();
        bank_stage(stage + BANK_STAGE_BUF, cur, cok, cs, BANK_STAGE_STEPS, in.T, in.ring, lane);
        cp_async_commit();
    }
    const uint64_t dXh = wg_desc(sW), dXl = wg_desc(sW + WG_TILE_BYTES), dU0h = wg_desc(sW + 2 * WG_TILE_BYTES),
                   dU0l = wg_desc(sW + 3 * WG_TILE_BYTES), dU1h = wg_desc(sW + 4 * WG_TILE_BYTES), dU1l = wg_desc(sW + 5 * WG_TILE_BYTES);
    constexpr uint64_t C6 = (6 * 256) >> 4;                  // descriptor offset of n-tile 6: the candidate's columns
    const int ra = w.ract, ac = w.act;
    int chunk = 0, cr = 0;
    float h[3][4] = {};

#pragma unroll 1
    for (int step = 0; step < in.T; ++step) {
        float xv[2][4];
        if (STAGE) {
            if (cr == 0) {
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
            if (cr + 1 == BANK_STAGE_STEPS) {
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
                const float* row = ok[hf] ? input_row(in, idx[hf], step) : nullptr;
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
        float acc[36];                                       // n-tile nt in acc[4 nt .. 4 nt + 3]: z 0..2, r 3..5, candidate 6..8
#pragma unroll
        for (int nt = 0; nt < MMA_NT; ++nt) {
            const float b0 = sb[8 * nt + 2 * t], b1 = sb[8 * nt + 2 * t + 1];
            acc[4 * nt] = b0; acc[4 * nt + 1] = b1; acc[4 * nt + 2] = b0; acc[4 * nt + 3] = b1;
        }
        uint32_t ah[4], al[4], ch[4] = {0u, 0u, 0u, 0u}, cl[4] = {0u, 0u, 0u, 0u};
        {
            uint32_t c2h[2], c2l[2];
            frag_f16(h, ah, al, c2h, c2l);
            ch[0] = c2h[0]; ch[1] = c2h[1]; cl[0] = c2l[0]; cl[1] = c2l[1];
        }
        // x part of all gates (lo.hi, hi.lo, hi.hi; z, r as n48 and the candidate as n24: an n24 inside an n72 accumulator
        // makes ptxas serialize every wgmma of the step), then h part of z and r
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
                for (int e = 0; e < 4; ++e) {
                    const float r = KERAS_ACT ? hard_sigmoid(acc[4 * (3 + nt) + e]) : apply_ract(acc[4 * (3 + nt) + e], ra);
                    rh[nt][e] = __fmul_rn(r, h[nt][e]);
                }
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
        // h = z h + (1 - z) a, rounded as in bank_scan
#pragma unroll
        for (int nt = 0; nt < 3; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float z = KERAS_ACT ? hard_sigmoid(acc[4 * nt + e]) : apply_ract(acc[4 * nt + e], ra);
                const float a = KERAS_ACT ? acc[4 * (6 + nt) + e] : apply_act(acc[4 * (6 + nt) + e], ac);
                h[nt][e] = __fmaf_rn(z, h[nt][e], __fmul_rn(__fsub_rn(1.f, z), a));
            }
    }
    if (STAGE) cp_async_wait<0>();
    const float* sWd = sb + 72;
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
        float part = 0.f;
#pragma unroll
        for (int nt = 0; nt < 3; ++nt) {
            part = fmaf(h[nt][2 * hf], sWd[8 * nt + 2 * t], part);
            part = fmaf(h[nt][2 * hf + 1], sWd[8 * nt + 2 * t + 1], part);
        }
        part += __shfl_xor_sync(0xffffffffu, part, 1);
        part += __shfl_xor_sync(0xffffffffu, part, 2);
        epilogue(part + w.bd, t == 0 && ok[hf], idx[hf], sid[hf], P.dp[0], P.o[0]);
    }
}

}  // namespace pb
