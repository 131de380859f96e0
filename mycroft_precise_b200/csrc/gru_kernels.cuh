// gru_kernels.cuh -- K2 (GRU window scan + Dense + sigmoid) fused with K3 (threshold decode,
// trigger debounce, detection count).
//
// Network: precise/model.py:77-82 -- GRU(H, activation='linear', Keras default
// recurrent_activation='hard_sigmoid', reset_after=False) + Dense(1,'sigmoid'), evaluated from
// h0 = 0 over all T = n_features rows on every update (precise/network_runner.py:148-153).
// Decode: precise/threshold_decoder.py:45-57.  Trigger: runner/precise_runner/runner.py:127-142.
//
// gru_small_kernel<H,F>: one thread per stream.  The whole weight set (8.2 KB at H=20, F=13) is a
//   __grid_constant__ kernel parameter, i.e. it sits in the constant bank and every FFMA takes
//   its weight as a constant operand: no weight loads at all, h/z/r stay in registers.
// gru_tiled_kernel: any H, F.  A CTA owns 64 streams; per step two register-tiled SGEMM phases
//   ([x,h] x [Wz|Wr], then [x,r*h] x Wh) with activations in shared memory and weights streamed
//   through L1/L2.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "mfcc_fast.cuh"      // smem_u32, mbarrier and bulk-copy helpers (staged projection blocks of the tensor-core scan)

namespace pb {

struct DecodeParams {
    const double* cd;        // cumulative distribution LUT
    int cd_len;
    int min_out, out_range;
    double center;
    double hot_threshold;    // 1.0 - sensitivity
    int trigger_level;
    int trigger_reset;       // -(8*2048) // chunk_bytes  (python floor division)
    int legacy_f64;          // pb_config.decode_legacy_f64
};

struct K2Out {
    float* raw;                      // [n] or null
    float* logit;                    // [n] or null
    double* conf;                    // [n] or null
    uint8_t* fired;                  // [n] or null
    unsigned long long* count;       // [1] or null
    int* trig;                       // [max_streams] or null => no trigger update
};

// Where row t of item i comes from.
struct K2In {
    const float* inputs;             // predict mode: [n][T][F_in] contiguous
    const float* ring;               // stream mode: [max_streams][ring_rows][row_stride]
    const long long* n_samples;      // stream mode: samples consumed (after this tick)
    const int* ids;                  // stream mode: item -> stream id (null = identity)
    int ring_rows, row_stride, window, hop;
    int T, F_base;                   // F_base = MFCC width (without deltas)
    int use_delta;
    const float* proj;               // non-null: cached input projections x.W + b, tile-major [ring_rows][proj_tiles] blocks of PROJ_BLOCK floats (see proj_off), same slots as ring
    int proj_tiles;                  // ceil(max_streams / 16)
    int used;                        // samples a frame needs before it is computed (min(window, n_fft)): tells which ring rows a tick has added
    int chunk;                       // samples added by this tick (to tell which window rows are new)
};

__device__ __forceinline__ float hard_sigmoid(float x) { return fminf(fmaxf(fmaf(0.2f, x, 0.5f), 0.f), 1.f); }
__device__ __forceinline__ float sigmoid32(float x) { return 1.f / (1.f + expf(-x)); }

template <int RACT>
__device__ __forceinline__ float ract(float x) { return RACT == 0 ? hard_sigmoid(x) : sigmoid32(x); }
template <int ACT>
__device__ __forceinline__ float act(float x) { return ACT == 0 ? x : tanhf(x); }

// ThresholdDecoder.decode on a float32 network output.  Runner.run hands the decoder an np.float32
// (network_runner.py:73-74, :94-95), so functions.asigmoid (functions.py:99-101) evaluates `1 / x - 1` in float32 under
// NumPy >= 2 promotion rules and only math.log in double; under NumPy 1.16 the same expression is float64
// (d.legacy_f64).  Everything after the logarithm is Python float (double) arithmetic in both cases.
__device__ __forceinline__ double decode_one(float raw, const DecodeParams& d) {
    const double r = (double)raw;
    if (raw == 1.0f || raw == 0.0f) return r;
    double cp;
    if (d.out_range == 0) {
        cp = r > (double)d.min_out ? 1.0 : 0.0;
    } else {
        const double t = d.legacy_f64 ? 1.0 / r - 1.0 : (double)__fsub_rn(__fdiv_rn(1.0f, raw), 1.0f);
        double lg = -log(t);                                           // functions.asigmoid
        double ratio = (lg - (double)d.min_out) / (double)d.out_range;
        ratio = fmin(fmax(ratio, 0.0), 1.0);
        int idx = (int)__dadd_rn(__dmul_rn(ratio, (double)(d.cd_len - 1)), 0.5);
        cp = d.cd[idx];
    }
    if (cp < d.center) return __dmul_rn(0.5, cp) / d.center;
    return __dadd_rn(0.5, __dmul_rn(0.5, cp - d.center) / (1.0 - d.center));
}

// Sigmoid + decode + trigger + count for item i (stream sid).  Called by every thread of the
// warp (valid = false for padding lanes) because the count is warp-aggregated.
__device__ __forceinline__ void epilogue(float logit, bool valid, long long i, int sid,
                                         const DecodeParams& d, const K2Out& o) {
    bool fired = false;
    if (valid) {
        float raw = sigmoid32(logit);
        if (o.logit) o.logit[i] = logit;
        if (o.raw) o.raw[i] = raw;
        if (o.conf || o.trig) {
            double conf = decode_one(raw, d);
            if (o.conf) o.conf[i] = conf;
            if (o.trig) {
                int a = o.trig[sid];
                const bool hot = conf > d.hot_threshold;
                if (hot || a < 0) {
                    a += 1;
                    fired = a > d.trigger_level;
                    if (fired || (hot && a < 0)) a = d.trigger_reset;
                } else if (a > 0) {
                    a -= 1;
                }
                o.trig[sid] = a;
                if (o.fired) o.fired[i] = fired ? 1 : 0;
            }
        }
    }
    if (o.count) {
        unsigned m = __ballot_sync(0xffffffffu, fired);
        if (m && (threadIdx.x & 31) == 0) atomicAdd(o.count, (unsigned long long)__popc(m));
    }
}

// Row pointer of window row t for item i, or nullptr for an all-zero row
// (rows before the stream's first frame: Listener.mfccs starts as zeros, network_runner.py:104).
__device__ __forceinline__ const float* ring_row(const K2In& in, int sid, long long released, int t) {
    long long k = released - in.T + t;
    if (k < 0) return nullptr;
    return in.ring + ((long long)sid * in.ring_rows + (int)(k % in.ring_rows)) * in.row_stride;
}

// Incremental form of ring_row for the scan kernels: one 64-bit modulo per stream instead of one per step.
struct RingCursor {
    const float* base;     // this stream's ring
    int slot;              // ring slot of window row 0 (valid once step >= lead)
    int lead;              // number of leading all-zero rows
    int rows, stride;
    __device__ __forceinline__ void init(const K2In& in, int sid, long long released) {
        const long long first = released - in.T;
        lead = first < 0 ? (int)(-first < in.T ? -first : in.T) : 0;
        long long m = first % in.ring_rows;
        if (m < 0) m += in.ring_rows;
        slot = (int)m;
        rows = in.ring_rows; stride = in.row_stride;
        base = in.ring + (long long)sid * in.ring_rows * in.row_stride;
    }
    // same window over the projection cache: next() returns the 16-stream block of this stream's tile at the step's slot
    // (blocks of `pblock` floats, slot-major); the row's position inside the block is proj_off(nt, sid & 15, t)
    __device__ __forceinline__ void init_proj(const K2In& in, int sid, long long released, int pblock) {
        init(in, sid, released);
        stride = in.proj_tiles * pblock;
        base = in.proj + (long long)(sid >> 4) * pblock;
    }
    // row of step t (call with t = 0, 1, 2, ... in order), nullptr for a zero row
    __device__ __forceinline__ const float* next(int t) {
        const float* r = t >= lead ? base + (long long)slot * stride : nullptr;
        slot = slot + 1 == rows ? 0 : slot + 1;
        return r;
    }
};

// ------------------------------------------------------------------------------------------------
template <int H, int F>
struct GruSmallW {
    float W[F][3 * H];
    float U[H][3 * H];
    float b[3 * H];
    float wd[H];
    float bd;
};

constexpr int K2_SMALL_THREADS = 128;
constexpr int K2_NS = 2;                       // streams per thread: every weight fetched feeds 2 FMAs

// dot product of column j of [W;U] (shared memory, transposed: Wt[j][0..K)) with [x | hv], for the
// K2_NS streams of this thread.  Weight loads are warp-uniform 16-byte broadcasts.
template <int H, int F, int KP>
__device__ __forceinline__ void gate_dot(const float (*Wt)[KP], int j, float bias, const float (&x)[K2_NS][F],
                                         const float (&hv)[K2_NS][H], float (&a)[K2_NS]) {
    // two partial sums per stream (even / odd k) double the number of independent FMA chains
    float a0[K2_NS], a1[K2_NS];
#pragma unroll
    for (int s = 0; s < K2_NS; ++s) { a0[s] = bias; a1[s] = 0.f; }
#pragma unroll
    for (int q = 0; q < KP / 4; ++q) {
        const float4 w = *reinterpret_cast<const float4*>(&Wt[j][4 * q]);
        const float wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int k = 4 * q + e;
            if (k < F + H) {
#pragma unroll
                for (int s = 0; s < K2_NS; ++s) {
                    const float vin = k < F ? x[s][k < F ? k : 0] : hv[s][k >= F ? k - F : 0];
                    if (e & 1) a1[s] = fmaf(vin, wv[e], a1[s]);
                    else a0[s] = fmaf(vin, wv[e], a0[s]);
                }
            }
        }
    }
#pragma unroll
    for (int s = 0; s < K2_NS; ++s) a[s] = a0[s] + a1[s];
}

// One thread owns K2_NS adjacent streams; h, z, r*h live in registers.  The weights sit in shared
// memory transposed -- column j of [W;U] is one contiguous row of KP = roundup4(F + H) floats -- and are
// fetched with warp-uniform (broadcast) 16-byte loads: with 2-way register blocking that is 9 LDS.128
// per 66 FFMA.
template <int H, int F, bool RING>
__global__ void __launch_bounds__(K2_SMALL_THREADS, 3)
gru_small_kernel(const __grid_constant__ GruSmallW<H, F> P, K2In in, long long n, DecodeParams dp, K2Out out) {
    constexpr int K = F + H, KP = (K + 3) & ~3;
    __shared__ __align__(16) float Wt[3 * H][KP];
    __shared__ float bs[3 * H];
    for (int e = threadIdx.x; e < 3 * H * KP; e += blockDim.x) {
        const int j = e / KP, k = e - j * KP;
        Wt[j][k] = k < F ? P.W[k][j] : (k < K ? P.U[k - F][j] : 0.f);
    }
    for (int e = threadIdx.x; e < 3 * H; e += blockDim.x) bs[e] = P.b[e];
    __syncthreads();

    const long long i0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * K2_NS;
    bool valid[K2_NS];
    int sid[K2_NS];
    long long released[K2_NS];
    RingCursor cur[K2_NS];
    float h[K2_NS][H];
#pragma unroll
    for (int s = 0; s < K2_NS; ++s) {
        valid[s] = i0 + s < n;
        sid[s] = 0; released[s] = 0;
#pragma unroll
        for (int j = 0; j < H; ++j) h[s][j] = 0.f;
        if (RING && valid[s]) {
            sid[s] = in.ids ? in.ids[i0 + s] : (int)(i0 + s);
            const long long ns = in.n_samples[sid[s]];
            released[s] = ns >= in.window ? (ns - in.window) / in.hop + 1 : 0;
            cur[s].init(in, sid[s], released[s]);
        }
    }
    if (valid[0]) {
#pragma unroll 1
        for (int t = 0; t < in.T; ++t) {
            float x[K2_NS][F];
#pragma unroll
            for (int s = 0; s < K2_NS; ++s) {
#pragma unroll
                for (int f = 0; f < F; ++f) x[s][f] = 0.f;
                if (!valid[s]) continue;
                if (RING) {
                    const float* row = cur[s].next(t);
                    if (row != nullptr) {
                        const float4* r4 = reinterpret_cast<const float4*>(row);   // rows: 16-byte aligned, padded to 4k floats
#pragma unroll
                        for (int q = 0; q < (F + 3) / 4; ++q) {
                            const float4 u = __ldg(r4 + q);
                            if (4 * q + 0 < F) x[s][4 * q + 0] = u.x;
                            if (4 * q + 1 < F) x[s][4 * q + 1] = u.y;
                            if (4 * q + 2 < F) x[s][4 * q + 2] = u.z;
                            if (4 * q + 3 < F) x[s][4 * q + 3] = u.w;
                        }
                    }
                } else {
                    const float* row = in.inputs + ((i0 + s) * in.T + t) * F;
#pragma unroll
                    for (int f = 0; f < F; ++f) x[s][f] = __ldg(row + f);
                }
            }
            float z[K2_NS][H], rh[K2_NS][H], a[K2_NS];
#pragma unroll
            for (int j = 0; j < H; ++j) {
                gate_dot<H, F, KP>(Wt, j, bs[j], x, h, a);
#pragma unroll
                for (int s = 0; s < K2_NS; ++s) z[s][j] = hard_sigmoid(a[s]);
            }
#pragma unroll
            for (int j = 0; j < H; ++j) {
                gate_dot<H, F, KP>(Wt, H + j, bs[H + j], x, h, a);
#pragma unroll
                for (int s = 0; s < K2_NS; ++s) rh[s][j] = hard_sigmoid(a[s]) * h[s][j];
            }
#pragma unroll
            for (int j = 0; j < H; ++j) {
                gate_dot<H, F, KP>(Wt, 2 * H + j, bs[2 * H + j], x, rh, a);
#pragma unroll
                for (int s = 0; s < K2_NS; ++s) z[s][j] = z[s][j] * h[s][j] + (1.f - z[s][j]) * a[s];   // linear candidate
            }
#pragma unroll
            for (int s = 0; s < K2_NS; ++s)
#pragma unroll
                for (int j = 0; j < H; ++j) h[s][j] = z[s][j];
        }
    }
#pragma unroll
    for (int s = 0; s < K2_NS; ++s) {
        float logit = P.bd;
#pragma unroll
        for (int j = 0; j < H; ++j) logit = fmaf(h[s][j], P.wd[j], logit);
        epilogue(logit, valid[s], i0 + s, sid[s], dp, out);
    }
}

// ------------------------------------------------------------------------------------------------
// Latency variant for small batches (BASELINE configs[1] and [4]): one WARP per stream.  Lane l < H owns
// hidden unit l for all three gates with its 3 x (F + H) weights in registers; h and r*h are exchanged
// with warp shuffles, so a step is ~2 x (H shuffles + a (F+H)-long FMA chain split 4 ways) instead of a
// thread walking all 3H x (F+H) products serially.
template <int H, int F, bool RING>
__global__ void __launch_bounds__(128)
gru_warp_kernel(const __grid_constant__ GruSmallW<H, F> P, K2In in, long long n, DecodeParams dp, K2Out out) {
    static_assert(H <= 32, "one lane per hidden unit");
    const int lane = threadIdx.x & 31;
    const long long i = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= n) return;                                   // whole warp exits together
    const int u = lane < H ? lane : 0;
    float wz[F + H], wr[F + H], wh[F + H];
#pragma unroll
    for (int k = 0; k < F; ++k) { wz[k] = P.W[k][u]; wr[k] = P.W[k][H + u]; wh[k] = P.W[k][2 * H + u]; }
#pragma unroll
    for (int k = 0; k < H; ++k) { wz[F + k] = P.U[k][u]; wr[F + k] = P.U[k][H + u]; wh[F + k] = P.U[k][2 * H + u]; }
    const float bz = P.b[u], br = P.b[H + u], bh = P.b[2 * H + u];
    int sid = 0;
    long long released = 0;
    if (RING) {
        sid = in.ids ? in.ids[i] : (int)i;
        const long long ns = in.n_samples[sid];
        released = ns >= in.window ? (ns - in.window) / in.hop + 1 : 0;
    }
    RingCursor cur;
    if (RING) cur.init(in, sid, released);
    // the whole window is fetched up front, one row per lane (T <= 32), so the scan itself never waits on memory:
    // step t takes its x_t from lane t with shuffles
    const bool prefetched = in.T <= 32;
    float xrow[F];
#pragma unroll
    for (int f = 0; f < F; ++f) xrow[f] = 0.f;
    if (prefetched) {
        const float* row = nullptr;
        if (lane < in.T) {
            if (RING) {
                const int t = lane;
                if (t >= cur.lead) { int sl = cur.slot + t; sl = sl >= cur.rows ? sl - cur.rows : sl; row = cur.base + sl * cur.stride; }
            } else {
                row = in.inputs + (i * in.T + lane) * F;
            }
        }
        if (row != nullptr) {
#pragma unroll
            for (int f = 0; f < F; ++f) xrow[f] = __ldg(row + f);
        }
    }
    float h = 0.f;
#pragma unroll 1
    for (int t = 0; t < in.T; ++t) {
        float x[F];
        if (prefetched) {
#pragma unroll
            for (int f = 0; f < F; ++f) x[f] = __shfl_sync(0xffffffffu, xrow[f], t);
        } else {
            const float* row = RING ? cur.next(t) : in.inputs + (i * in.T + t) * F;
#pragma unroll
            for (int f = 0; f < F; ++f) x[f] = row ? __ldg(row + f) : 0.f;          // same address in every lane: broadcast
        }
        float az[4] = {bz, 0.f, 0.f, 0.f}, ar[4] = {br, 0.f, 0.f, 0.f}, ah[4] = {bh, 0.f, 0.f, 0.f};
#pragma unroll
        for (int f = 0; f < F; ++f) {
            az[f & 3] = fmaf(x[f], wz[f], az[f & 3]);
            ar[f & 3] = fmaf(x[f], wr[f], ar[f & 3]);
            ah[f & 3] = fmaf(x[f], wh[f], ah[f & 3]);
        }
#pragma unroll
        for (int k = 0; k < H; ++k) {
            const float hk = __shfl_sync(0xffffffffu, h, k);
            az[k & 3] = fmaf(hk, wz[F + k], az[k & 3]);
            ar[k & 3] = fmaf(hk, wr[F + k], ar[k & 3]);
        }
        const float z = hard_sigmoid((az[0] + az[1]) + (az[2] + az[3]));
        const float rh = hard_sigmoid((ar[0] + ar[1]) + (ar[2] + ar[3])) * h;
#pragma unroll
        for (int k = 0; k < H; ++k) {
            const float v = __shfl_sync(0xffffffffu, rh, k);
            ah[k & 3] = fmaf(v, wh[F + k], ah[k & 3]);
        }
        const float hh = (ah[0] + ah[1]) + (ah[2] + ah[3]);
        h = z * h + (1.f - z) * hh;
    }
    float part = lane < H ? h * P.wd[u] : 0.f;
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) part += __shfl_xor_sync(0xffffffffu, part, d);
    // lane 0 finishes; other lanes take part in the ballot with valid = false
    epilogue(part + P.bd, lane == 0, i, sid, dp, out);
}

// ------------------------------------------------------------------------------------------------
// Tensor-core variant of the small network (H <= 24, F <= 16): the per-step products [x_t | h] x [W;U]
// run on the warp-level tensor-core path (mma.sync m16n8k8, TF32 inputs, fp32 accumulate) with the
// 3xTF32 split (a = a_hi + a_lo, b = b_hi + b_lo; a_lo b_hi + a_hi b_lo + a_hi b_hi) so that the result
// keeps fp32-level accuracy (parity tolerance 1e-5).  A warp owns 16*MB streams (rows of the A operand);
// h, z, r*h stay in accumulator-fragment layout in registers for all 29 steps.
//
// Contraction-index trick: the k index of an MMA is only a summation label, so the hidden units are
// assigned to k slots in the order the accumulator fragment already holds them (thread t of a quad owns
// units 8*tile + 2t, 2t+1).  The weight fragments are permuted once on the host to match; turning h
// (C layout) into the next step's A operand then needs no shuffle at all.
constexpr int PROJ_COLS = 72;        // padded gate columns of the fragment layout: 24 * gate + unit
constexpr int PROJ_STRIDE = 60;      // projection values per frame: 20 * gate + unit (the padding units are not stored)
constexpr int PROJ_BLOCK = 16 * PROJ_STRIDE;    // floats of one (slot, 16-stream tile) block of the cache
constexpr int PROJ_FRAMES_PER_CTA = 4;
// Layout of a block: the scan's accumulator-fragment order, so that one LDG.64 of a warp (n-tile nt, row half hf; lane = 4 g + t reads
// columns 2t, 2t + 1 of row g + 8 hf) is 256 contiguous bytes when the tile's 16 streams sit at the same ring slot -- 2 cache lines
// per request instead of 8 scattered 32-byte sectors (round 2: the row-major cache kept the scan bound by L1 line requests,
// 144 per warp and step).  Full n-tiles (nt % 3 != 2, 8 units) first: [6][16 rows][4 t][2]; then the half n-tiles (units 16..19 of
// a gate, t < 2): [3][16 rows][2 t][2].
__host__ __device__ __forceinline__ int proj_off(int nt, int r16, int t) {
    return nt % 3 != 2 ? ((nt / 3) * 2 + nt % 3) * 128 + r16 * 8 + 2 * t : 768 + (nt / 3) * 64 + r16 * 4 + 2 * t;
}

constexpr int MMA_KT = 5;            // k tiles: 2 for x (F <= 16), 3 for h (H <= 24)
constexpr int MMA_NT = 9;            // n tiles: z, r, h gates x 3 tiles of 8 units
constexpr int MMA_MB = 2;            // row blocks of 16 streams per warp
constexpr int MMA_THREADS = 128;

struct GruMmaW {
    const float4* bfrag;             // [MMA_KT][MMA_NT][32 lanes] (b0_hi, b1_hi, b0_lo, b1_lo)
    const float* bias;               // [3][24] padded per gate
    const float* wd;                 // [24] padded
    float bd;
};

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// 3xTF32: d += a_lo b_hi + a_hi b_lo + a_hi b_hi for a group of NG n-tiles and MB row blocks.  The three
// terms are issued as three sweeps over the group so that consecutive MMAs never target the same
// accumulator (dependent distance NG * MB instructions).
template <int NG, int MB>
__device__ __forceinline__ void mma3_group(float (*acc)[MMA_NT][4], int nt0, const uint32_t (*ah)[4], const uint32_t (*al)[4],
                                           const float4 (&w)[NG]) {
#pragma unroll
    for (int q = 0; q < NG; ++q)
#pragma unroll
        for (int mb = 0; mb < MB; ++mb) mma_tf32(acc[mb][nt0 + q], al[mb], __float_as_uint(w[q].x), __float_as_uint(w[q].y));
#pragma unroll
    for (int q = 0; q < NG; ++q)
#pragma unroll
        for (int mb = 0; mb < MB; ++mb) mma_tf32(acc[mb][nt0 + q], ah[mb], __float_as_uint(w[q].z), __float_as_uint(w[q].w));
#pragma unroll
    for (int q = 0; q < NG; ++q)
#pragma unroll
        for (int mb = 0; mb < MB; ++mb) mma_tf32(acc[mb][nt0 + q], ah[mb], __float_as_uint(w[q].x), __float_as_uint(w[q].y));
}

// hi = a with the 13 low mantissa bits cleared (what the tensor core reads anyway), lo = a - hi (exact in
// fp32; the tensor core truncates it to TF32 again, leaving a relative error <= 2^-21 per product).
// One LOP3 + one FADD per element instead of two cvt.rna.tf32 (which issue on the quarter-rate XU pipe).
__device__ __forceinline__ void split_tf32(const float (&v)[4], uint32_t (&hi)[4], uint32_t (&lo)[4]) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        hi[e] = __float_as_uint(v[e]) & 0xffffe000u;
        lo[e] = __float_as_uint(v[e] - __uint_as_float(hi[e]));
    }
}

// PROJ (stream mode): the input projection x_t.[Wz|Wr|Wh] + b of every frame was computed once when the frame was
// produced (input_proj_kernel) and sits in the ring next to the MFCC row, so the scan only runs the recurrent products:
// 162 instead of 270 HMMA per step on the pipe that bounds this kernel.
// MB = row blocks of 16 streams per warp.  2 halves the weight-fragment traffic per MMA; 1 halves the tile (and the
// registers: 5 instead of 3 CTAs per SM), which matters for the tail of the grid -- see launch_gru.
// STAGED (PROJ, MB = 1): a warp whose 16 streams form one aligned tile at one ring slot (the common case: streams in lock step)
// reads a step's projections as ONE contiguous 3840-byte block -- fetched by a bulk async copy (cp.async.bulk, SASS UBLKCP) into
// a per-warp double buffer two steps ahead, completion on an mbarrier; the accumulators then start from conflict-free LDS.64.
// No register and no scoreboard wait sits between DRAM and the MMAs.  Other warps (ragged ids / ages) keep the LDG path.
constexpr int K2_STAGE_BYTES = PROJ_BLOCK * 4;                                       // 3840
constexpr int K2_STAGED_SMEM = (MMA_THREADS / 32) * (2 * K2_STAGE_BYTES + 16);      // + two mbarriers per warp

template <int H, int F, bool RING, bool PROJ, int MB = MMA_MB, bool STAGED = false>
__global__ void __launch_bounds__(MMA_THREADS, MB == 1 ? (STAGED ? 4 : 5) : 3)
gru_mma_kernel(GruMmaW W, K2In in, long long n, DecodeParams dp, K2Out out) {
    static_assert(H <= 24 && F <= 16, "tile counts are fixed");
    static_assert(!STAGED || (PROJ && RING && MB == 1), "staging serves the stream scan over cached projections");
    extern __shared__ __align__(128) unsigned char k2_stage_raw[];
    __shared__ float4 sB[MMA_KT * MMA_NT * 32];
    __shared__ float sBias[3 * 24];
    __shared__ float sWd[24];
    for (int e = threadIdx.x; e < MMA_KT * MMA_NT * 32; e += blockDim.x) sB[e] = __ldg(W.bfrag + e);
    for (int e = threadIdx.x; e < 72; e += blockDim.x) sBias[e] = __ldg(W.bias + e);
    for (int e = threadIdx.x; e < 24; e += blockDim.x) sWd[e] = __ldg(W.wd + e);
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    const long long base = ((long long)blockIdx.x * (MMA_THREADS / 32) + warp) * (16 * MB);
    if (base >= n) return;
    // rows of this thread: stream (mb, hf) = base + 16 mb + g + 8 hf
    long long idx[MB][2];
    int sid[MB][2];
    long long rel[MB][2];
    RingCursor cur[MB][2];
    bool ok[MB][2];
#pragma unroll
    for (int mb = 0; mb < MB; ++mb)
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            idx[mb][hf] = base + 16 * mb + g + 8 * hf;
            ok[mb][hf] = idx[mb][hf] < n;
            sid[mb][hf] = 0; rel[mb][hf] = 0;
            if (RING && ok[mb][hf]) {
                sid[mb][hf] = in.ids ? in.ids[idx[mb][hf]] : (int)idx[mb][hf];
                const long long ns = in.n_samples[sid[mb][hf]];
                rel[mb][hf] = ns >= in.window ? (ns - in.window) / in.hop + 1 : 0;
                if (PROJ) cur[mb][hf].init_proj(in, sid[mb][hf], rel[mb][hf], PROJ_BLOCK);
                else cur[mb][hf].init(in, sid[mb][hf], rel[mb][hf]);
            }
        }
    // h in accumulator layout: hreg[mb][tile][e], e = (row g: units 2t, 2t+1; row g+8: units 2t, 2t+1) of tile
    float hreg[MB][3][4];
#pragma unroll
    for (int mb = 0; mb < MB; ++mb)
#pragma unroll
        for (int nt = 0; nt < 3; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) hreg[mb][nt][e] = 0.f;

    // ---- STAGED: is this warp's tile uniform?  Then its projection blocks arrive by bulk copies.
    bool staged = false;
    float* stg = nullptr;
    unsigned long long* sbar = nullptr;
    const float* sblock = nullptr;                      // block of the tile at slot 0
    int s_slot0 = 0, s_lead = 0, s_rows = 1;
    long long s_stride = 0;
    uint32_t s_ph0 = 0, s_ph1 = 0;
    if constexpr (STAGED) {
        stg = reinterpret_cast<float*>(k2_stage_raw + warp * 2 * K2_STAGE_BYTES);
        sbar = reinterpret_cast<unsigned long long*>(k2_stage_raw + (MMA_THREADS / 32) * 2 * K2_STAGE_BYTES) + 2 * warp;
        const int sid0 = __shfl_sync(0xffffffffu, sid[0][0], 0);
        const int sl0 = __shfl_sync(0xffffffffu, cur[0][0].slot, 0), ld0 = __shfl_sync(0xffffffffu, cur[0][0].lead, 0);
        const bool same = ok[0][0] && ok[0][1] && (sid0 & 15) == 0 && sid[0][0] == sid0 + g && sid[0][1] == sid0 + g + 8 &&
                          cur[0][0].slot == sl0 && cur[0][1].slot == sl0 && cur[0][0].lead == ld0 && cur[0][1].lead == ld0;
        staged = __all_sync(0xffffffffu, same);
        if (staged) {
            s_slot0 = sl0; s_lead = ld0; s_rows = cur[0][0].rows; s_stride = cur[0][0].stride; sblock = cur[0][0].base;
            if (lane == 0) { mbar_init(&sbar[0], 1); mbar_init(&sbar[1], 1); fence_mbar_init(); }
            __syncwarp();
        }
    }
    auto stage_issue = [&](int st) {                    // lane 0: the block of step st into buffer st & 1
        int sl = s_slot0 + st;
        if (sl >= s_rows) sl -= s_rows;
        unsigned long long* bar = &sbar[st & 1];
        mbar_expect_tx(bar, (uint32_t)K2_STAGE_BYTES);
        bulk_g2s(stg + (st & 1) * PROJ_BLOCK, sblock + (long long)sl * s_stride, (uint32_t)K2_STAGE_BYTES, bar);
    };
    if (STAGED && staged && lane == 0) {
        if (s_lead < in.T) stage_issue(s_lead);
        if (s_lead + 1 < in.T) stage_issue(s_lead + 1);
    }

#pragma unroll 1
    for (int step = 0; step < in.T; ++step) {
        float acc[MB][MMA_NT][4];
        if (STAGED && staged) {
            // ---- accumulators from the staged block (bias for the rows before the stream's first frame)
            const bool real = step >= s_lead;
            const float* blk = stg + (step & 1) * PROJ_BLOCK;
            if (real) {
                if (step & 1) { mbar_wait(&sbar[1], s_ph1); s_ph1 ^= 1u; } else { mbar_wait(&sbar[0], s_ph0); s_ph0 ^= 1u; }
            }
#pragma unroll
            for (int mb = 0; mb < MB; ++mb)
#pragma unroll
                for (int hf = 0; hf < 2; ++hf)
#pragma unroll
                    for (int nt = 0; nt < MMA_NT; ++nt) {
                        float2 v;
                        if (!real) v = make_float2(sBias[8 * nt + 2 * t], sBias[8 * nt + 2 * t + 1]);
                        else if (nt % 3 != 2 || t < 2) v = *reinterpret_cast<const float2*>(blk + proj_off(nt, g + 8 * hf, t));
                        else v = make_float2(0.f, 0.f);
                        acc[mb][nt][2 * hf] = v.x; acc[mb][nt][2 * hf + 1] = v.y;
                    }
        } else if (PROJ) {
            // ---- accumulators start from the cached projection (bias included); rows before the stream's first frame: bias
#pragma unroll
            for (int mb = 0; mb < MB; ++mb)
#pragma unroll
                for (int hf = 0; hf < 2; ++hf) {
                    const float* row = ok[mb][hf] ? cur[mb][hf].next(step) : nullptr;
#pragma unroll
                    for (int nt = 0; nt < MMA_NT; ++nt) {
                        float2 v;
                        if (row == nullptr) v = make_float2(sBias[8 * nt + 2 * t], sBias[8 * nt + 2 * t + 1]);
                        else if (nt % 3 != 2 || t < 2) v = __ldg(reinterpret_cast<const float2*>(row + proj_off(nt, sid[mb][hf] & 15, t)));
                        else v = make_float2(0.f, 0.f);                  // padding units 20..23 of a gate: not stored
                        acc[mb][nt][2 * hf] = v.x; acc[mb][nt][2 * hf + 1] = v.y;
                    }
                }
        } else {
            // ---- A fragments of x_t: a0 = (row g, k 2t), a1 = (row g+8, k 2t), a2 = (row g, k 2t+1), a3 = (row g+8, k 2t+1)
            uint32_t xh[MB][2][4], xl[MB][2][4];
#pragma unroll
            for (int mb = 0; mb < MB; ++mb) {
                float xv[2][2][2];                               // [kt][hf][j]
#pragma unroll
                for (int hf = 0; hf < 2; ++hf) {
                    const float* row = nullptr;
                    if (ok[mb][hf]) row = RING ? cur[mb][hf].next(step) : in.inputs + (idx[mb][hf] * in.T + step) * F;
#pragma unroll
                    for (int kt = 0; kt < 2; ++kt)
#pragma unroll
                        for (int j = 0; j < 2; ++j) {
                            const int f = 8 * kt + 2 * t + j;
                            xv[kt][hf][j] = (row != nullptr && f < F) ? __ldg(row + f) : 0.f;
                        }
                }
#pragma unroll
                for (int kt = 0; kt < 2; ++kt) {
                    const float v[4] = {xv[kt][0][0], xv[kt][1][0], xv[kt][0][1], xv[kt][1][1]};
                    split_tf32(v, xh[mb][kt], xl[mb][kt]);
                }
            }
            // ---- accumulators start from the bias (column 2t + j of tile nt)
#pragma unroll
            for (int nt = 0; nt < MMA_NT; ++nt) {
                const float b0 = sBias[8 * nt + 2 * t], b1 = sBias[8 * nt + 2 * t + 1];
#pragma unroll
                for (int mb = 0; mb < MB; ++mb) { acc[mb][nt][0] = b0; acc[mb][nt][1] = b1; acc[mb][nt][2] = b0; acc[mb][nt][3] = b1; }
            }
            // ---- x part for all three gates
#pragma unroll
            for (int kt = 0; kt < 2; ++kt) {
                uint32_t ah[MB][4], al[MB][4];
#pragma unroll
                for (int mb = 0; mb < MB; ++mb)
#pragma unroll
                    for (int e = 0; e < 4; ++e) { ah[mb][e] = xh[mb][kt][e]; al[mb][e] = xl[mb][kt][e]; }
#pragma unroll
                for (int ng = 0; ng < MMA_NT; ng += 3) {
                    float4 w[3];
#pragma unroll
                    for (int q = 0; q < 3; ++q) w[q] = sB[(kt * MMA_NT + ng + q) * 32 + lane];
                    mma3_group<3, MB>(acc, ng, ah, al, w);
                }
            }
        }
        // ---- h part for z and r
#pragma unroll
        for (int kt = 0; kt < 3; ++kt) {
            uint32_t ah[MB][4], al[MB][4];
#pragma unroll
            for (int mb = 0; mb < MB; ++mb) {
                const float v[4] = {hreg[mb][kt][0], hreg[mb][kt][2], hreg[mb][kt][1], hreg[mb][kt][3]};
                split_tf32(v, ah[mb], al[mb]);
            }
#pragma unroll
            for (int ng = 0; ng < 6; ng += 3) {
                float4 w[3];
#pragma unroll
                for (int q = 0; q < 3; ++q) w[q] = sB[((2 + kt) * MMA_NT + ng + q) * 32 + lane];
                mma3_group<3, MB>(acc, ng, ah, al, w);
            }
        }
        // ---- gates; r * h becomes the A operand of the candidate product
#pragma unroll
        for (int kt = 0; kt < 3; ++kt) {
            uint32_t ah[MB][4], al[MB][4];
#pragma unroll
            for (int mb = 0; mb < MB; ++mb) {
                float rh[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) rh[e] = hard_sigmoid(acc[mb][3 + kt][e]) * hreg[mb][kt][e];
                const float v[4] = {rh[0], rh[2], rh[1], rh[3]};
                split_tf32(v, ah[mb], al[mb]);
            }
            {
                float4 w[3];
#pragma unroll
                for (int q = 0; q < 3; ++q) w[q] = sB[((2 + kt) * MMA_NT + 6 + q) * 32 + lane];
                mma3_group<3, MB>(acc, 6, ah, al, w);
            }
        }
#pragma unroll
        for (int mb = 0; mb < MB; ++mb)
#pragma unroll
            for (int nt = 0; nt < 3; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float z = hard_sigmoid(acc[mb][nt][e]);
                    hreg[mb][nt][e] = z * hreg[mb][nt][e] + (1.f - z) * acc[mb][6 + nt][e];      // linear candidate
                }
        if (STAGED && staged && step >= s_lead && step + 2 < in.T) {     // this step's buffer has been consumed by every lane: refill it
            __syncwarp();
            if (lane == 0) stage_issue(step + 2);
        }
    }
    // ---- Dense(1): per-thread partial over its 6 units per row, reduced over the quad
#pragma unroll
    for (int mb = 0; mb < MB; ++mb)
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            float part = 0.f;
#pragma unroll
            for (int nt = 0; nt < 3; ++nt) {
                part = fmaf(hreg[mb][nt][2 * hf], sWd[8 * nt + 2 * t], part);
                part = fmaf(hreg[mb][nt][2 * hf + 1], sWd[8 * nt + 2 * t + 1], part);
            }
            part += __shfl_xor_sync(0xffffffffu, part, 1);
            part += __shfl_xor_sync(0xffffffffu, part, 2);
            epilogue(part + W.bd, t == 0 && ok[mb][hf], idx[mb][hf], sid[mb][hf], dp, out);
        }
}

// ------------------------------------------------------------------------------------------------
// ------------------------------------------------------------------------------------------------
// The steady-state stream scan over cached projections with the recurrent products in fp16 x 3 (hi / lo split of both operands,
// fp32 accumulate: a_lo b_hi + a_hi b_lo + a_hi b_hi) on mma.sync m16n8k16 / m16n8k8: one k16 + one k8 MMA per n-tile and pass
// cover the 24 (padded) hidden units that the TF32 kernel above needs three k8 MMAs for -- half the tensor-pipe time, which is
// what bounds the scan once its loads are staged (ncu: math_pipe_throttle).  Hidden units sit in the k index in natural order
// (thread t of a quad holds units 8 tile + 2t, 2t + 1 in its accumulators = the (2t, 2t + 1) and (2t + 8, 2t + 9) k pairs of the
// A fragment), so h turns into the next step's A operand with two F2FP packs per n-tile and no data movement.
// Accuracy: pieces of 11 bits each, 22 bits per product like 3xTF32 (CPU emulation on the default network: 7.6e-8 vs 4.7e-8).
struct GruMma16W {
    const uint4* bfrag;              // [2 k-tiles][MMA_NT][32 lanes] (b0_hi, b1_hi, b0_lo, b1_lo) as half2; k-tile 1 uses b0 only (units 16..23)
    const uint4* xfrag;              // [MMA_NT][32 lanes]: the input weights (features 0..15 as one k16 fragment), same packing
    const float* bias;               // [3][24] padded per gate
    const float* wd;                 // [24] padded
    float bd;
};

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

// The kernel also keeps the cache itself: before the scan, every warp projects the frames this tick has added for its 16 streams
// (x . [Wz|Wr|Wh] + b, one k16 MMA per n-tile and pass) and writes them into the cache blocks -- the separate projection
// kernel of the other variants (39 us per tick) is not launched on this path.
template <int H, int F, int CTAS = 4>
__global__ void __launch_bounds__(MMA_THREADS, CTAS)
gru_mma16_kernel(GruMma16W W, K2In in, long long n, DecodeParams dp, K2Out out) {
    static_assert(H <= 24 && F <= 16, "tile counts are fixed");
    extern __shared__ __align__(128) unsigned char k2_stage_raw[];
    __shared__ uint4 sB[2 * MMA_NT * 32];
    __shared__ uint4 sX[MMA_NT * 32];
    for (int e = threadIdx.x; e < MMA_NT * 32; e += blockDim.x) sX[e] = __ldg(W.xfrag + e);
    __shared__ float sBias[3 * 24];
    __shared__ float sWd[24];
    for (int e = threadIdx.x; e < 2 * MMA_NT * 32; e += blockDim.x) sB[e] = __ldg(W.bfrag + e);
    for (int e = threadIdx.x; e < 72; e += blockDim.x) sBias[e] = __ldg(W.bias + e);
    for (int e = threadIdx.x; e < 24; e += blockDim.x) sWd[e] = __ldg(W.wd + e);
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    const long long base = ((long long)blockIdx.x * (MMA_THREADS / 32) + warp) * 16;
    if (base >= n) return;
    long long idx[2];
    int sid[2];
    RingCursor cur[2];
    bool ok[2];
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
        idx[hf] = base + g + 8 * hf;
        ok[hf] = idx[hf] < n;
        sid[hf] = 0;
        if (ok[hf]) {
            sid[hf] = in.ids ? in.ids[idx[hf]] : (int)idx[hf];
            const long long ns = in.n_samples[sid[hf]];
            cur[hf].init_proj(in, sid[hf], ns >= in.window ? (ns - in.window) / in.hop + 1 : 0, PROJ_BLOCK);
        }
    }
    float hreg[3][4];
#pragma unroll
    for (int nt = 0; nt < 3; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) hreg[nt][e] = 0.f;

    // ---- the frames this tick has added to the ring (cf. input_proj_kernel): project them and store them into the cache
    {
        int slot0[2], cnt[2];
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            slot0[hf] = 0; cnt[hf] = 0;
            if (ok[hf]) {
                const long long n1 = in.n_samples[sid[hf]], n0 = n1 - in.chunk;
                const long long c0 = n0 >= in.used ? (n0 - in.used) / in.hop + 1 : 0, c1 = n1 >= in.used ? (n1 - in.used) / in.hop + 1 : 0;
                slot0[hf] = (int)(c0 % in.ring_rows); cnt[hf] = (int)(c1 - c0);
            }
        }
        int maxc = max(cnt[0], cnt[1]);
#pragma unroll
        for (int d = 16; d >= 1; d >>= 1) maxc = max(maxc, __shfl_xor_sync(0xffffffffu, maxc, d));
        float* pw = const_cast<float*>(in.proj);
#pragma unroll 1
        for (int j = 0; j < maxc; ++j) {
            float xv[2][4];
            float* blk[2];
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
                blk[hf] = nullptr;
                xv[hf][0] = xv[hf][1] = xv[hf][2] = xv[hf][3] = 0.f;
                if (j < cnt[hf]) {
                    int sl = slot0[hf] + j;
                    if (sl >= in.ring_rows) sl -= in.ring_rows;
                    const float* row = in.ring + ((long long)sid[hf] * in.ring_rows + sl) * in.row_stride;
                    blk[hf] = pw + ((long long)sl * in.proj_tiles + (sid[hf] >> 4)) * PROJ_BLOCK;
                    if (2 * t < F) xv[hf][0] = row[2 * t];
                    if (2 * t + 1 < F) xv[hf][1] = row[2 * t + 1];
                    if (2 * t + 8 < F) xv[hf][2] = row[2 * t + 8];
                    if (2 * t + 9 < F) xv[hf][3] = row[2 * t + 9];
                }
            }
            uint32_t ah[4], al[4];
            split_f16(xv[0][0], xv[0][1], ah[0], al[0]);
            split_f16(xv[1][0], xv[1][1], ah[1], al[1]);
            split_f16(xv[0][2], xv[0][3], ah[2], al[2]);
            split_f16(xv[1][2], xv[1][3], ah[3], al[3]);
#pragma unroll 1
            for (int ng = 0; ng < MMA_NT; ng += 3) {
                float a3[3][4];
                uint4 w[3];
#pragma unroll
                for (int q = 0; q < 3; ++q) {
                    const float b0 = sBias[8 * (ng + q) + 2 * t], b1 = sBias[8 * (ng + q) + 2 * t + 1];
                    a3[q][0] = b0; a3[q][1] = b1; a3[q][2] = b0; a3[q][3] = b1;
                    w[q] = sX[(ng + q) * 32 + lane];
                }
#pragma unroll
                for (int q = 0; q < 3; ++q) mma_f16_k16(a3[q], al, w[q].x, w[q].y);
#pragma unroll
                for (int q = 0; q < 3; ++q) mma_f16_k16(a3[q], ah, w[q].z, w[q].w);
#pragma unroll
                for (int q = 0; q < 3; ++q) mma_f16_k16(a3[q], ah, w[q].x, w[q].y);
#pragma unroll
                for (int hf = 0; hf < 2; ++hf)
                    if (blk[hf] != nullptr) {
#pragma unroll
                        for (int q = 0; q < 3; ++q)
                            if (q < 2 || t < 2)
                                *reinterpret_cast<float2*>(blk[hf] + proj_off(ng + q, sid[hf] & 15, t)) = make_float2(a3[q][2 * hf], a3[q][2 * hf + 1]);
                    }
            }
        }
        // the scan reads these rows through the async proxy (bulk copies) or with plain loads: order them after the stores
        asm volatile("fence.proxy.async.global;" ::: "memory");
        __threadfence_block();
        __syncwarp();
    }

    // ---- uniform tile: projection blocks by bulk copy (see gru_mma_kernel<.., STAGED>)
    float* stg = reinterpret_cast<float*>(k2_stage_raw + warp * 2 * K2_STAGE_BYTES);
    unsigned long long* sbar = reinterpret_cast<unsigned long long*>(k2_stage_raw + (MMA_THREADS / 32) * 2 * K2_STAGE_BYTES) + 2 * warp;
    const int sid0 = __shfl_sync(0xffffffffu, sid[0], 0);
    const int sl0 = __shfl_sync(0xffffffffu, cur[0].slot, 0), ld0 = __shfl_sync(0xffffffffu, cur[0].lead, 0);
    const bool same = ok[0] && ok[1] && (sid0 & 15) == 0 && sid[0] == sid0 + g && sid[1] == sid0 + g + 8 &&
                      cur[0].slot == sl0 && cur[1].slot == sl0 && cur[0].lead == ld0 && cur[1].lead == ld0;
    const bool staged = __all_sync(0xffffffffu, same);
    const float* sblock = cur[0].base;
    const int s_rows = cur[0].rows;
    const long long s_stride = cur[0].stride;
    uint32_t s_ph0 = 0, s_ph1 = 0;
    auto stage_issue = [&](int st) {
        int sl = sl0 + st;
        if (sl >= s_rows) sl -= s_rows;
        unsigned long long* bar = &sbar[st & 1];
        mbar_expect_tx(bar, (uint32_t)K2_STAGE_BYTES);
        bulk_g2s(stg + (st & 1) * PROJ_BLOCK, sblock + (long long)sl * s_stride, (uint32_t)K2_STAGE_BYTES, bar);
    };
    if (staged) {
        if (lane == 0) { mbar_init(&sbar[0], 1); mbar_init(&sbar[1], 1); fence_mbar_init(); }
        __syncwarp();
        if (lane == 0) {
            if (ld0 < in.T) stage_issue(ld0);
            if (ld0 + 1 < in.T) stage_issue(ld0 + 1);
        }
    }

#pragma unroll 1
    for (int step = 0; step < in.T; ++step) {
        float acc[MMA_NT][4];
        if (staged) {
            const bool real = step >= ld0;
            const float* blk = stg + (step & 1) * PROJ_BLOCK;
            if (real) {
                if (step & 1) { mbar_wait(&sbar[1], s_ph1); s_ph1 ^= 1u; } else { mbar_wait(&sbar[0], s_ph0); s_ph0 ^= 1u; }
            }
#pragma unroll
            for (int hf = 0; hf < 2; ++hf)
#pragma unroll
                for (int nt = 0; nt < MMA_NT; ++nt) {
                    float2 v;
                    if (!real) v = make_float2(sBias[8 * nt + 2 * t], sBias[8 * nt + 2 * t + 1]);
                    else if (nt % 3 != 2 || t < 2) v = *reinterpret_cast<const float2*>(blk + proj_off(nt, g + 8 * hf, t));
                    else v = make_float2(0.f, 0.f);
                    acc[nt][2 * hf] = v.x; acc[nt][2 * hf + 1] = v.y;
                }
        } else {
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
                const float* row = ok[hf] ? cur[hf].next(step) : nullptr;
#pragma unroll
                for (int nt = 0; nt < MMA_NT; ++nt) {
                    float2 v;
                    if (row == nullptr) v = make_float2(sBias[8 * nt + 2 * t], sBias[8 * nt + 2 * t + 1]);
                    else if (nt % 3 != 2 || t < 2) v = __ldg(reinterpret_cast<const float2*>(row + proj_off(nt, sid[hf] & 15, t)));
                    else v = make_float2(0.f, 0.f);
                    acc[nt][2 * hf] = v.x; acc[nt][2 * hf + 1] = v.y;
                }
            }
        }
        // ---- h part for z and r
        {
            uint32_t ah[4], al[4], ch[2], cl[2];
            frag_f16(hreg, ah, al, ch, cl);
            mma3_f16(acc, 0, ah, al, ch, cl, sB, lane);
            mma3_f16(acc, 3, ah, al, ch, cl, sB, lane);
        }
        // ---- gates; r * h is the A operand of the candidate product
        {
            float rh[3][4];
#pragma unroll
            for (int nt = 0; nt < 3; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) rh[nt][e] = hard_sigmoid(acc[3 + nt][e]) * hreg[nt][e];
            uint32_t ah[4], al[4], ch[2], cl[2];
            frag_f16(rh, ah, al, ch, cl);
            mma3_f16(acc, 6, ah, al, ch, cl, sB, lane);
        }
#pragma unroll
        for (int nt = 0; nt < 3; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float z = hard_sigmoid(acc[nt][e]);
                hreg[nt][e] = z * hreg[nt][e] + (1.f - z) * acc[6 + nt][e];      // linear candidate
            }
        if (staged && step >= ld0 && step + 2 < in.T) {          // this step's buffer has been consumed by every lane: refill it
            __syncwarp();
            if (lane == 0) stage_issue(step + 2);
        }
    }
    // ---- Dense(1): per-thread partial over its 6 units per row, reduced over the quad
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
        float part = 0.f;
#pragma unroll
        for (int nt = 0; nt < 3; ++nt) {
            part = fmaf(hreg[nt][2 * hf], sWd[8 * nt + 2 * t], part);
            part = fmaf(hreg[nt][2 * hf + 1], sWd[8 * nt + 2 * t + 1], part);
        }
        part += __shfl_xor_sync(0xffffffffu, part, 1);
        part += __shfl_xor_sync(0xffffffffu, part, 2);
        epilogue(part + W.bd, t == 0 && ok[hf], idx[hf], sid[hf], dp, out);
    }
}

// Cached input projection (default network, stream mode): a = b + x . [Wz|Wr|Wh] (60 floats per frame) is kept in a second
// ring with the same slot numbering as the MFCC ring.  A steady-state scan reads 29 x 240 B of it per stream -- the scan is
// bound by that traffic, which is why the rows are stored compact (no padding units) and apart from the MFCC rows.
// input_proj_kernel fills the rows of a tick's new frames; input_proj_all_kernel refreshes every row after the cache was
// invalidated.

// Per-tick projection of the frames a tick has just produced, on the tensor cores: a warp takes 32 new frames as the rows
// of two m16 blocks and runs the 3xTF32 x-part MMAs (2 k-tiles x 9 n-tiles) once per frame instead of once per scan step.
// Register-lean (n-tiles in groups of three) so that one or two waves cover a whole tick: the kernel is latency-bound
// (two dependent scattered reads per frame).  Items are ordered j-major (item = j * n + i): warps stay converged when the
// streams run in lock step.
constexpr int PROJ_THREADS = 128;

template <int F>
__global__ void __launch_bounds__(PROJ_THREADS, 6)
input_proj_kernel(const float4* __restrict__ bfrag, const float* __restrict__ bias, const long long* __restrict__ n_samples,
                  const int* __restrict__ ids, int n, int chunk, int need, int hop, int max_new,
                  const float* __restrict__ ring, int ring_rows, int row_stride, float* __restrict__ proj, int proj_tiles) {
    __shared__ float4 sB[2 * MMA_NT * 32];
    __shared__ float sBias[PROJ_COLS];
    for (int e = threadIdx.x; e < 2 * MMA_NT * 32; e += blockDim.x) sB[e] = __ldg(bfrag + e);
    for (int e = threadIdx.x; e < PROJ_COLS; e += blockDim.x) sBias[e] = __ldg(bias + e);
    __syncthreads();
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const long long items = (long long)n * max_new;
    const long long base = ((long long)blockIdx.x * (PROJ_THREADS / 32) + (threadIdx.x >> 5)) * 32;
    if (base >= items) return;
    const float* rows[MMA_MB][2];
    float* prow[MMA_MB][2];
    int r16[MMA_MB][2];
#pragma unroll
    for (int mb = 0; mb < MMA_MB; ++mb)
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            rows[mb][hf] = nullptr; prow[mb][hf] = nullptr; r16[mb][hf] = 0;
            const long long item = base + 16 * mb + g + 8 * hf;
            if (item < items) {
                const int j = (int)(item / n);
                const long long i = item - (long long)j * n;
                const int sid = ids ? ids[i] : (int)i;
                const long long n1 = n_samples[sid], n0 = n1 - chunk;
                const long long c0 = n0 >= need ? (n0 - need) / hop + 1 : 0, c1 = n1 >= need ? (n1 - need) / hop + 1 : 0;
                if (j < c1 - c0) {
                    const int slot = (int)((c0 + j) % ring_rows);
                    rows[mb][hf] = ring + ((long long)sid * ring_rows + slot) * row_stride;
                    prow[mb][hf] = proj + ((long long)slot * proj_tiles + (sid >> 4)) * PROJ_BLOCK;
                    r16[mb][hf] = sid & 15;
                }
            }
        }
    uint32_t ah[2][MMA_MB][4], al[2][MMA_MB][4];
#pragma unroll
    for (int kt = 0; kt < 2; ++kt)
#pragma unroll
        for (int mb = 0; mb < MMA_MB; ++mb) {
            float v[4];
#pragma unroll
            for (int hf = 0; hf < 2; ++hf)
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const int f = 8 * kt + 2 * t + j;
                    v[2 * j + hf] = (rows[mb][hf] != nullptr && f < F) ? rows[mb][hf][f] : 0.f;     // a0,a1 = rows (g, g+8), k = 2t ; a2,a3: k = 2t+1
                }
            split_tf32(v, ah[kt][mb], al[kt][mb]);
        }
#pragma unroll 1
    for (int ng = 0; ng < MMA_NT; ng += 3) {
        float acc[MMA_MB][3][4];
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            const float b0 = sBias[8 * (ng + q) + 2 * t], b1 = sBias[8 * (ng + q) + 2 * t + 1];
#pragma unroll
            for (int mb = 0; mb < MMA_MB; ++mb) { acc[mb][q][0] = b0; acc[mb][q][1] = b1; acc[mb][q][2] = b0; acc[mb][q][3] = b1; }
        }
#pragma unroll
        for (int kt = 0; kt < 2; ++kt) {
            float4 w[3];
#pragma unroll
            for (int q = 0; q < 3; ++q) w[q] = sB[(kt * MMA_NT + ng + q) * 32 + lane];
#pragma unroll
            for (int q = 0; q < 3; ++q)
#pragma unroll
                for (int mb = 0; mb < MMA_MB; ++mb) mma_tf32(acc[mb][q], al[kt][mb], __float_as_uint(w[q].x), __float_as_uint(w[q].y));
#pragma unroll
            for (int q = 0; q < 3; ++q)
#pragma unroll
                for (int mb = 0; mb < MMA_MB; ++mb) mma_tf32(acc[mb][q], ah[kt][mb], __float_as_uint(w[q].z), __float_as_uint(w[q].w));
#pragma unroll
            for (int q = 0; q < 3; ++q)
#pragma unroll
                for (int mb = 0; mb < MMA_MB; ++mb) mma_tf32(acc[mb][q], ah[kt][mb], __float_as_uint(w[q].x), __float_as_uint(w[q].y));
        }
#pragma unroll
        for (int mb = 0; mb < MMA_MB; ++mb)
#pragma unroll
            for (int hf = 0; hf < 2; ++hf)
                if (prow[mb][hf] != nullptr) {
#pragma unroll
                    for (int q = 0; q < 3; ++q)
                        if (q < 2 || t < 2)                          // ng is a multiple of 3: q == 2 is the half-empty tile of the gate
                            *reinterpret_cast<float2*>(prow[mb][hf] + proj_off(ng + q, r16[mb][hf], t)) = make_float2(acc[mb][q][2 * hf], acc[mb][q][2 * hf + 1]);
                }
    }
}

// Same projection for EVERY ring row of every stream: run once after the weights change or after ticks that skipped the
// per-tick projection (small batches served by the warp-per-stream kernel), so that cached projections are always valid.
template <int F>
__global__ void __launch_bounds__(64 * PROJ_FRAMES_PER_CTA)
input_proj_all_kernel(const float* __restrict__ wx, const float* __restrict__ bias, long long total_rows,
                      const float* __restrict__ ring, int ring_rows, int row_stride, float* __restrict__ proj, int proj_tiles) {
    __shared__ float sW[F * PROJ_COLS];
    for (int e = threadIdx.x; e < F * PROJ_COLS; e += blockDim.x) sW[e] = __ldg(wx + e);
    __syncthreads();
    const int c = threadIdx.x & 63, fl = threadIdx.x >> 6;          // c: stored column 20 * gate + unit
    if (c >= PROJ_STRIDE) return;
    const int col = c + 4 * (c / 20);                                // padded column 24 * gate + unit
    for (long long r = (long long)blockIdx.x * PROJ_FRAMES_PER_CTA + fl; r < total_rows; r += (long long)gridDim.x * PROJ_FRAMES_PER_CTA) {
        const float* row = ring + r * row_stride;
        float a = __ldg(bias + col);
#pragma unroll
        for (int f = 0; f < F; ++f) a = fmaf(row[f], sW[f * PROJ_COLS + col], a);
        const long long sid = r / ring_rows;
        const int slot = (int)(r - sid * ring_rows), unit = c % 20, nt = 3 * (c / 20) + unit / 8;
        proj[((long long)slot * proj_tiles + (sid >> 4)) * PROJ_BLOCK + proj_off(nt, (int)(sid & 15), (unit & 7) >> 1) + (unit & 1)] = a;
    }
}

// ------------------------------------------------------------------------------------------------
// Generic tiled kernel.  wcat = [kernel; recurrent] as one [(F_in + H)][3H] row-major matrix.
constexpr int K2_TILE_THREADS = 256;
constexpr int K2_TILE_STREAMS = 64;     // 8 warps x 8 streams
constexpr int K2_COLS_PER_THREAD = 8;   // columns tx + 32 c

struct GruTiledW {
    const float* wcat;   // [(F_in + H)][3H]
    const float* bias;   // [3H]
    const float* wd;     // [H]
    float bd;
    int H, F_in;
    int act, ract;
};

__device__ __forceinline__ float apply_ract(float x, int kind) { return kind == 0 ? hard_sigmoid(x) : sigmoid32(x); }
__device__ __forceinline__ float apply_act(float x, int kind) { return kind == 0 ? x : tanhf(x); }

// acc[s][c] += sum_k A[k][8*warp + s] * Wcat[row0 + k][col(c)] for k in [0, K)
__device__ __forceinline__ void tile_mac(float (&acc)[8][K2_COLS_PER_THREAD], const float* __restrict__ A,
                                         const float* __restrict__ wrow, int ldw, int K, int col0, int ncols_total, int warp, int lane) {
    for (int k = 0; k < K; ++k) {
        const float4 a0 = *reinterpret_cast<const float4*>(A + k * K2_TILE_STREAMS + 8 * warp);
        const float4 a1 = *reinterpret_cast<const float4*>(A + k * K2_TILE_STREAMS + 8 * warp + 4);
        const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float* w = wrow + (long long)k * ldw;
#pragma unroll
        for (int c = 0; c < K2_COLS_PER_THREAD; ++c) {
            int j = col0 + lane + 32 * c;
            float wv = j < ncols_total ? __ldg(w + j) : 0.f;
#pragma unroll
            for (int s = 0; s < 8; ++s) acc[s][c] = fmaf(av[s], wv, acc[s][c]);
        }
    }
}

template <bool RING>
__global__ void __launch_bounds__(K2_TILE_THREADS)
gru_tiled_kernel(GruTiledW W, K2In in, long long n, DecodeParams dp, K2Out out) {
    extern __shared__ __align__(16) float sm[];
    const int H = W.H, F = W.F_in, H3 = 3 * W.H;
    float* X = sm;                               // [F][64]
    float* Hs = X + F * K2_TILE_STREAMS;         // [H][64]   (rows F.. of the [x,h] activation matrix)
    float* RH = Hs + H * K2_TILE_STREAMS;        // [H][64]
    float* Z = RH + H * K2_TILE_STREAMS;         // [H][64]
    __shared__ int s_sid[K2_TILE_STREAMS];
    __shared__ long long s_rel[K2_TILE_STREAMS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long base = (long long)blockIdx.x * K2_TILE_STREAMS;
    if (threadIdx.x < K2_TILE_STREAMS) {
        long long i = base + threadIdx.x;
        int sid = 0; long long rel = 0;
        if (RING && i < n) {
            sid = in.ids ? in.ids[i] : (int)i;
            long long ns = in.n_samples[sid];
            rel = ns >= in.window ? (ns - in.window) / in.hop + 1 : 0;
        }
        s_sid[threadIdx.x] = sid; s_rel[threadIdx.x] = rel;
    }
    for (int e = threadIdx.x; e < H * K2_TILE_STREAMS; e += blockDim.x) Hs[e] = 0.f;
    __syncthreads();
    const int Fb = in.F_base;
    for (int t = 0; t < in.T; ++t) {
        // ---- stage x_t (and deltas) for the 64 streams: X[f][b]
        for (int e = threadIdx.x; e < F * K2_TILE_STREAMS; e += blockDim.x) {
            int f = e / K2_TILE_STREAMS, b = e - f * K2_TILE_STREAMS;   // conflict-free smem store; row reuse hits L1
            long long i = base + b;
            float v = 0.f;
            if (i < n) {
                if (RING) {
                    int fb = f < Fb ? f : f - Fb;
                    const float* row = ring_row(in, s_sid[b], s_rel[b], t);
                    float cur = row ? row[fb] : 0.f;
                    if (f < Fb) v = cur;
                    else if (t > 0) {                      // add_deltas: delta[0] = 0
                        const float* prow = ring_row(in, s_sid[b], s_rel[b], t - 1);
                        v = cur - (prow ? prow[fb] : 0.f);
                    }
                } else {
                    v = __ldg(in.inputs + (i * in.T + t) * F + f);
                }
            }
            X[f * K2_TILE_STREAMS + b] = v;
        }
        __syncthreads();
        // ---- phase 1: z, r  (columns [0, 2H))
        for (int col0 = 0; col0 < 2 * H; col0 += 32 * K2_COLS_PER_THREAD) {
            float acc[8][K2_COLS_PER_THREAD];
#pragma unroll
            for (int c = 0; c < K2_COLS_PER_THREAD; ++c) {
                int j = col0 + lane + 32 * c;
                float bj = j < 2 * H ? __ldg(W.bias + j) : 0.f;
#pragma unroll
                for (int s = 0; s < 8; ++s) acc[s][c] = bj;
            }
            tile_mac(acc, X, W.wcat, H3, F, col0, 2 * H, warp, lane);
            tile_mac(acc, Hs, W.wcat + (long long)F * H3, H3, H, col0, 2 * H, warp, lane);
#pragma unroll
            for (int c = 0; c < K2_COLS_PER_THREAD; ++c) {
                int j = col0 + lane + 32 * c;
                if (j < 2 * H) {
#pragma unroll
                    for (int s = 0; s < 8; ++s) {
                        float g = apply_ract(acc[s][c], W.ract);
                        int b = 8 * warp + s;
                        if (j < H) Z[j * K2_TILE_STREAMS + b] = g;
                        else RH[(j - H) * K2_TILE_STREAMS + b] = g * Hs[(j - H) * K2_TILE_STREAMS + b];
                    }
                }
            }
        }
        __syncthreads();
        // ---- phase 2: candidate + state update (columns [2H, 3H))
        for (int col0 = 0; col0 < H; col0 += 32 * K2_COLS_PER_THREAD) {
            float acc[8][K2_COLS_PER_THREAD];
#pragma unroll
            for (int c = 0; c < K2_COLS_PER_THREAD; ++c) {
                int j = col0 + lane + 32 * c;
                float bj = j < H ? __ldg(W.bias + 2 * H + j) : 0.f;
#pragma unroll
                for (int s = 0; s < 8; ++s) acc[s][c] = bj;
            }
            tile_mac(acc, X, W.wcat + 2 * H, H3, F, col0, H, warp, lane);
            tile_mac(acc, RH, W.wcat + (long long)F * H3 + 2 * H, H3, H, col0, H, warp, lane);
#pragma unroll
            for (int c = 0; c < K2_COLS_PER_THREAD; ++c) {
                int j = col0 + lane + 32 * c;
                if (j < H) {
#pragma unroll
                    for (int s = 0; s < 8; ++s) {
                        int b = 8 * warp + s;
                        float z = Z[j * K2_TILE_STREAMS + b], hp = Hs[j * K2_TILE_STREAMS + b];
                        Hs[j * K2_TILE_STREAMS + b] = z * hp + (1.f - z) * apply_act(acc[s][c], W.act);
                    }
                }
            }
        }
        __syncthreads();
    }
    // ---- Dense(1) + epilogue: warps 0,1 own the 64 streams
    if (warp < 2) {
        int b = threadIdx.x;
        long long i = base + b;
        float logit = W.bd;
        for (int j = 0; j < H; ++j) logit = fmaf(Hs[j * K2_TILE_STREAMS + b], __ldg(W.wd + j), logit);
        epilogue(logit, i < n, i, s_sid[b], dp, out);
    }
}

// K3 alone (pb_decode)
__global__ void decode_kernel(const float* __restrict__ raw, long long n, DecodeParams dp, double* __restrict__ conf) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) conf[i] = decode_one(raw[i], dp);
}

}  // namespace pb
