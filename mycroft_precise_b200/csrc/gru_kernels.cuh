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
#include <cuda_runtime.h>
#include <stdint.h>

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
    const uint8_t* route;            // [max_streams] per-stream model masks (pb_set_stream_models) or null => every stream scored
    unsigned route_bit;              // this model's bit of route[sid]
};

// Where row t of item i comes from.  Predict mode (!RING) reads row starts[i] + t of `inputs`, rows row_stride floats apart:
// pb_predict's [n][T][F_in] windows (starts null: item i starts at row i * T, row_stride = F_in), or a recorded corpus's
// frame rows (pb_score_corpus: one start row per window, rows of the MFCC width padded to 4, use_delta taken within the
// window).  The union keeps K2In, and with it every stream-tick kernel's parameter block, the size it had.
struct K2In {
    const float* inputs;             // predict mode: window rows (see above)
    const float* ring;               // stream mode: [max_streams][ring_rows][row_stride]
    union {
        const long long* n_samples;  // stream mode: samples consumed (after this tick)
        const long long* starts;     // predict mode: first row of item i's window, or null
    };
    const int* ids;                  // stream mode: item -> stream id (null = identity)
    int ring_rows, row_stride, window, hop;
    int T, F_base;                   // F_base = MFCC width (without deltas)
    int use_delta;
};

// Predict mode: row t of item i's window.
__device__ __forceinline__ const float* input_row(const K2In& in, long long i, int t) {
    return in.inputs + ((in.starts ? in.starts[i] : i * in.T) + t) * (long long)in.row_stride;
}

// Predict mode, column f of row t of item i: with use_delta (corpus windows of F_base columns) column f >= F_base is the
// delta of column f - F_base against row t - 1, 0 on row 0 (add_deltas within the window, network_runner.py:150-151).
__device__ __forceinline__ float input_value(const K2In& in, long long i, int t, int f) {
    const float* row = input_row(in, i, t);
    if (!in.use_delta || f < in.F_base) return __ldg(row + f);
    const int fb = f - in.F_base;
    return t > 0 ? __ldg(row + fb) - __ldg(row + fb - in.row_stride) : 0.f;
}

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
// warp (valid = false for padding lanes) because the count is warp-aggregated.  ROUTE: a stream whose route mask lacks the
// model's bit is not scored: no output written (route_kernel fills its NaN), no trigger update, not counted.  The check leaves
// every kernel's registers as they were except gru_small_kernel's spills, so that kernel alone has instantiations without it.
template <bool ROUTE = true>
__device__ __forceinline__ void epilogue(float logit, bool valid, long long i, int sid,
                                         const DecodeParams& d, const K2Out& o) {
    if (ROUTE && valid && o.route && !(o.route[sid] & o.route_bit)) valid = false;
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
    // row of step t (call with t = 0, 1, 2, ... in order), nullptr for a zero row
    __device__ __forceinline__ const float* next(int t) {
        const float* r = t >= lead ? base + (long long)slot * stride : nullptr;
        slot = slot + 1 == rows ? 0 : slot + 1;
        return r;
    }
    // row of step t in any order (t < T <= rows: the window wraps the ring at most once), nullptr for a zero row
    __device__ __forceinline__ const float* at(int t) const {
        if (t < lead) return nullptr;
        const int s = slot + t;
        return base + (long long)(s >= rows ? s - rows : s) * stride;
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
template <int H, int F, bool RING, bool ROUTE = false>
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
                    const float* row = input_row(in, i0 + s, t);
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
        epilogue<ROUTE>(logit, valid[s], i0 + s, sid[s], dp, out);
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
                row = input_row(in, i, lane);
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
            const float* row = RING ? cur.next(t) : input_row(in, i, t);
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
// Warp-level tensor-core (mma.sync) building blocks of the tensor-core scans: gru_bank.cuh and gru_wide.cuh.
constexpr int MMA_NT = 9;            // n tiles of the fused family: z, r, h gates x 3 tiles of 8 units
constexpr int MMA_THREADS = 128;

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
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
                    v = input_value(in, i, t, f);
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
