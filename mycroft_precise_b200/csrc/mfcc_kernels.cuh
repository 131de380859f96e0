// mfcc_kernels.cuh -- K1: PCM -> power spectrum -> mel -> log -> DCT (MFCC).
//
// Two entry kernels share the device code:
//   mfcc_batch_kernel   stateless: whole buffers [n_streams][L] -> [n_streams][n_frames][n_out]
//                       (vectorize_raw, precise/vectorization.py:46-50)
//   mfcc_stream_kernel  stateful tick: appends one chunk per stream, computes the frames that
//                       became computable, writes them into the per-stream MFCC ring and keeps
//                       the unconsumed PCM tail (Listener.update_vectors,
//                       precise/network_runner.py:125-146)
//
// Phase A (FFT, fft512.cuh): a warp transforms two frames at a time (16 lanes per frame) and
// leaves scaled power spectra in a shared-memory tile [<=32 frames][257].
// Phase B (mel/log/DCT): one thread per frame walks the 257 bins once.  Bin k lies in exactly one
// grid segment i = [g_i, g_i+1); it feeds the rising edge of filter i with weight w_rise[k] and
// the falling edge of filter i-1 with weight w_fall[k] (sonopy.filterbanks), so
// mel_j = rise(seg j) + fall(seg j+1).  Then log(max(.,eps)), the DCT-II(ortho) rows and the
// c0 := log(sum power) replacement (sonopy.mfcc_spec).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "fft512.cuh"

namespace pb {

constexpr int K1_THREADS = 128;
constexpr int K1_WARPS = K1_THREADS / 32;
constexpr int K1_TILE = 32;              // frames per round
constexpr int K1_PSTRIDE = 257;          // odd: thread-per-frame reads are bank-conflict free
constexpr int K1_STREAMS_PER_CTA = 32;   // stream kernel: streams per tile
constexpr float K1_EPS = 2.220446049250313e-16f;   // np.finfo(float).eps, sonopy.safe_log

struct MelTables {
    const float* w_rise;      // [n_bins]
    const float* w_fall;      // [n_bins]
    const int* grid;          // [n_filt + 2]
    const float* dct;         // [n_out][n_filt]
    const float2* tw_stage;   // [16][16]  (cos, -sin)(2 pi n2 k1 / 256)
    const float2* tw_post;    // [16]      (cos, +sin)(2 pi k1 / 512)
    int n_bins, n_filt, n_out;
    int mels_only;            // Vectorizer.mels: emit log-mels, no DCT / c0
    int n_fft;                // 512: register FFT (fft512.cuh); other powers of two <= 512: fft_any_power below
    const float2* tw_any;     // [n_fft / 2]  (cos, -sin)(2 pi k / n_fft)
};

// Where the `used` samples of one frame live: sample i is p0[i] for i < len0, else p1[i - len0];
// samples >= used are zero (window shorter than n_fft).
template <typename T>
struct FrameSrc {
    const T* p0;
    const T* p1;
    int len0;
    int used;
};

__device__ __forceinline__ float to_f(int16_t v) { return (float)v; }
__device__ __forceinline__ float to_f(float v) { return v; }

// packed complex element m = samples (2m, 2m+1)
template <typename T, bool PAIRS>
__device__ __forceinline__ cpx load_elem(const FrameSrc<T>& s, int m) {
    cpx r;
    int i = 2 * m;
    if (PAIRS) {   // len0, used even and both pointers pair-aligned: a pair never straddles
        if (i >= s.used) return {0.f, 0.f};
        const T* p = (i < s.len0) ? s.p0 + i : s.p1 + (i - s.len0);
        if (sizeof(T) == 2) {
            int v = __ldg(reinterpret_cast<const int*>(p));
            r.x = (float)(short)(v & 0xffff);
            r.y = (float)(short)(v >> 16);
        } else {
            float2 v = __ldg(reinterpret_cast<const float2*>(p));
            r.x = v.x; r.y = v.y;
        }
        return r;
    }
    r.x = (i < s.used) ? to_f(__ldg((i < s.len0) ? s.p0 + i : s.p1 + (i - s.len0))) : 0.f;
    ++i;
    r.y = (i < s.used) ? to_f(__ldg((i < s.len0) ? s.p0 + i : s.p1 + (i - s.len0))) : 0.f;
    return r;
}

// Any power-of-two n_fft <= 1024 (the reference lets n_fft be configured, precise/params.py:49; scratch: n_fft float2): a whole warp transforms
// one frame with a plain radix-2 shared-memory FFT (real input as complex), then writes the scaled power bins.  Slow path.
template <typename T>
__device__ __forceinline__ void fft_any_power(const FrameSrc<T>& s, int n_fft, const float2* __restrict__ tw, float2* scratch,
                                              float* P, float scale, int lane) {
    const int lg = 31 - __clz(n_fft);
    for (int i = lane; i < n_fft; i += 32) {
        float v = 0.f;
        if (i < s.used) v = to_f(__ldg(i < s.len0 ? s.p0 + i : s.p1 + (i - s.len0)));
        scratch[__brev((unsigned)i) >> (32 - lg)] = make_float2(v, 0.f);
    }
    __syncwarp();
    for (int len = 2; len <= n_fft; len <<= 1) {
        const int hl = len >> 1, step = n_fft / len;
        for (int b = lane; b < n_fft / 2; b += 32) {
            const int grp = b / hl, k = b - grp * hl, i0 = grp * len + k, i1 = i0 + hl;
            const float2 w = __ldg(tw + k * step), a = scratch[i0], c = scratch[i1];
            const float vr = fmaf(c.x, w.x, -c.y * w.y), vi = fmaf(c.x, w.y, c.y * w.x);
            scratch[i0] = make_float2(a.x + vr, a.y + vi);
            scratch[i1] = make_float2(a.x - vr, a.y - vi);
        }
        __syncwarp();
    }
    for (int k = lane; k <= n_fft / 2; k += 32) { const float2 a = scratch[k]; P[k] = fmaf(a.x, a.x, a.y * a.y) * scale; }
    __syncwarp();
}

// Per-CTA copy of the small tables (broadcast reads in phase B).
constexpr int K1_MAX_BINS = 513;          // n_fft <= 1024
constexpr int K1_PSTRIDE_BIG = 513;       // power-row stride for n_fft = 1024 (rows and FFT scratch then live in the dynamic tail, see k1_big_smem)
constexpr size_t k1_big_smem = (size_t)32 * K1_PSTRIDE_BIG * sizeof(float) + (size_t)4 * 1024 * sizeof(float2);   // K1_TILE rows + K1_WARPS scratches
constexpr int K1_MAX_FILT = 64;
struct K1Tables {
    float2 w[K1_MAX_BINS + 3];                 // (w_rise, w_fall) per bin
    int grid[K1_MAX_FILT + 2];
    float* dct;                                // [n_out][n_filt], in the dynamic tail of the CTA's shared memory
};

__device__ __forceinline__ void load_tables(K1Tables& s, const MelTables& t, float* dct_smem) {
    if (threadIdx.x == 0) s.dct = dct_smem;
    for (int k = threadIdx.x; k < t.n_bins; k += blockDim.x) s.w[k] = make_float2(__ldg(t.w_rise + k), __ldg(t.w_fall + k));
    for (int k = threadIdx.x; k < t.n_filt + 2; k += blockDim.x) s.grid[k] = __ldg(t.grid + k);
    if (!t.mels_only)
        for (int k = threadIdx.x; k < t.n_out * t.n_filt; k += blockDim.x) dct_smem[k] = __ldg(t.dct + k);
}

// Phase B for one frame: P = power row in shared memory (its head is overwritten with the log-mels),
// out = n_out floats (row_pad floats are written when PADDED: the destination row is 16-byte aligned
// and padded to a multiple of 4 floats).
template <bool PADDED>
__device__ __forceinline__ void mel_log_dct(float* P, const K1Tables& tb, const MelTables& t, float* __restrict__ out) {
    const int nb = t.n_bins;
    const float* dct = tb.dct;
    float tot0 = 0.f, tot1 = 0.f;
    const int g0 = tb.grid[0];
    for (int k = 0; k < g0 && k < nb; ++k) tot0 += P[k];
    float rise_prev = 0.f;
    for (int i = 0; i <= t.n_filt; ++i) {
        const int lo = tb.grid[i];
        int hi = tb.grid[i + 1];
        hi = hi < nb ? hi : nb;
        float r0 = 0.f, f0 = 0.f, r1 = 0.f, f1 = 0.f, r2 = 0.f, f2 = 0.f, r3 = 0.f, f3 = 0.f;
        int k = lo;
        for (; k + 3 < hi; k += 4) {
            const float p0 = P[k], p1 = P[k + 1], p2 = P[k + 2], p3 = P[k + 3];
            const float2 w0 = tb.w[k], w1 = tb.w[k + 1], w2 = tb.w[k + 2], w3 = tb.w[k + 3];
            tot0 += p0 + p2; tot1 += p1 + p3;
            r0 = fmaf(w0.x, p0, r0); f0 = fmaf(w0.y, p0, f0);
            r1 = fmaf(w1.x, p1, r1); f1 = fmaf(w1.y, p1, f1);
            r2 = fmaf(w2.x, p2, r2); f2 = fmaf(w2.y, p2, f2);
            r3 = fmaf(w3.x, p3, r3); f3 = fmaf(w3.y, p3, f3);
        }
        for (; k < hi; ++k) {
            const float p0 = P[k];
            const float2 w0 = tb.w[k];
            tot0 += p0;
            r0 = fmaf(w0.x, p0, r0); f0 = fmaf(w0.y, p0, f0);
        }
        if (i > 0) P[i - 1] = logf(fmaxf(rise_prev + ((f0 + f1) + (f2 + f3)), K1_EPS));   // grid[i+1] >= i+1: slot already consumed
        rise_prev = (r0 + r1) + (r2 + r3);
    }
    for (int k = tb.grid[t.n_filt + 1]; k < nb; ++k) tot0 += P[k];
    if (t.mels_only) {
        for (int j = 0; j < t.n_out; ++j) out[j] = P[j];
        return;
    }
    const float c0 = logf(fmaxf(tot0 + tot1, K1_EPS));
    if (PADDED) {
        // rows of 4 outputs, stored as float4
        for (int c4 = 0; c4 < t.n_out; c4 += 4) {
            float a[4] = {0.f, 0.f, 0.f, 0.f};
            for (int j = 0; j < t.n_filt; ++j) {
                const float m = P[j];
#pragma unroll
                for (int q = 0; q < 4; ++q)
                    if (c4 + q < t.n_out) a[q] = fmaf(dct[(c4 + q) * t.n_filt + j], m, a[q]);
            }
            if (c4 == 0) a[0] = c0;
            *reinterpret_cast<float4*>(out + c4) = make_float4(a[0], a[1], a[2], a[3]);
        }
    } else {
        out[0] = c0;
        for (int c = 1; c < t.n_out; ++c) {
            const float* d = dct + c * t.n_filt;
            float a0 = 0.f, a1 = 0.f;
            int j = 0;
            for (; j + 1 < t.n_filt; j += 2) { a0 = fmaf(d[j], P[j], a0); a1 = fmaf(d[j + 1], P[j + 1], a1); }
            if (j < t.n_filt) a0 = fmaf(d[j], P[j], a0);
            out[c] = a0 + a1;
        }
    }
}

struct K1Smem {
    float power[K1_TILE * K1_PSTRIDE];
    float2 xch[K1_WARPS * 2 * XCH_ELEMS];
    K1Tables tab;
};

// ------------------------------------------------------------------------------------------------
// Stateless batch kernel.  Global frame g = stream * n_frames + f.
template <typename T, bool PAIRS>
__global__ void __launch_bounds__(K1_THREADS, 4)
mfcc_batch_kernel(const T* __restrict__ pcm, long long samples_per_stream, long long n_frames_per_stream,
                  long long total_frames, int hop, int used, float scale, MelTables tab,
                  float* __restrict__ out) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    K1Smem& sm = *reinterpret_cast<K1Smem*>(smem_raw);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, l16 = lane & 15, half = lane >> 4;
    FftLaneConst lc;
    load_lane_const(lc, tab.tw_stage, tab.tw_post, l16);
    float2* xch = sm.xch + (warp * 2 + half) * XCH_ELEMS;
    load_tables(sm.tab, tab, reinterpret_cast<float*>(smem_raw + sizeof(K1Smem)));
    // n_fft = 1024: power rows (513 bins) and the warp FFT's scratch (1024 float2) do not fit the static arrays; they follow the DCT table
    const bool big = tab.n_fft > 512;
    unsigned char* big_base = smem_raw + ((sizeof(K1Smem) + (size_t)tab.n_out * tab.n_filt * sizeof(float) + 15) & ~(size_t)15);
    float* const power = big ? reinterpret_cast<float*>(big_base) : sm.power;
    const int ps = big ? K1_PSTRIDE_BIG : K1_PSTRIDE;
    float2* const xany = big ? reinterpret_cast<float2*>(big_base + (size_t)K1_TILE * K1_PSTRIDE_BIG * sizeof(float)) + warp * 1024 : sm.xch + warp * 2 * XCH_ELEMS;
    __syncthreads();
    const long long n_tiles = (total_frames + K1_TILE - 1) / K1_TILE;
    for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const long long g_base = tile * K1_TILE;
        // ---- phase A: 32 frames, 8 per pass over the 4 warps
        if (tab.n_fft != 512) {
#pragma unroll 1
            for (int slot = warp; slot < K1_TILE; slot += K1_WARPS) {           // generic n_fft: one frame per warp at a time
                const long long g = g_base + slot;
                if (g >= total_frames) break;
                const long long s = g / n_frames_per_stream, f = g - s * n_frames_per_stream;
                FrameSrc<T> src;
                src.p0 = pcm + s * samples_per_stream + f * hop;
                src.p1 = src.p0; src.len0 = used; src.used = used;
                fft_any_power<T>(src, tab.n_fft, tab.tw_any, xany, power + slot * ps, scale, lane);
            }
        } else
#pragma unroll 1
        for (int pass = 0; pass < K1_TILE / (K1_WARPS * 2); ++pass) {
            const int slot = pass * (K1_WARPS * 2) + warp * 2 + half;
            const long long g = g_base + slot;
            const bool active = g < total_frames;
            cpx z[16];
            if (active) {
                long long s = g / n_frames_per_stream, f = g - s * n_frames_per_stream;
                FrameSrc<T> src;
                src.p0 = pcm + s * samples_per_stream + f * hop;
                src.p1 = src.p0; src.len0 = used; src.used = used;
#pragma unroll
                for (int n1 = 0; n1 < 16; ++n1) z[n1] = load_elem<T, PAIRS>(src, 16 * n1 + l16);
            } else {
#pragma unroll
                for (int n1 = 0; n1 < 16; ++n1) z[n1] = {0.f, 0.f};
            }
            fft512_power(z, lc, xch, sm.power + slot * K1_PSTRIDE, scale, l16, active);
        }
        __syncthreads();
        // ---- phase B: thread per frame
        if (threadIdx.x < K1_TILE) {
            const long long g = g_base + threadIdx.x;
            if (g < total_frames) mel_log_dct<false>(power + threadIdx.x * ps, sm.tab, tab, out + g * tab.n_out);
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------
// Per-stream streaming state (device arrays owned by the handle).
struct StreamState {
    long long* n_samples;     // [max_streams] samples consumed so far
    int16_t* tail;            // [max_streams][tail_cap] unconsumed samples a later frame still needs
    float* ring;              // [max_streams][ring_rows][row_stride] MFCC rows, slot = frame index % ring_rows
    int tail_cap, ring_rows, row_stride;
};

__host__ __device__ __forceinline__ long long frames_ready(long long n, int need, int hop) {
    return n >= need ? (n - need) / hop + 1 : 0;
}

// Ragged tick (pb_update_ragged): where item i's samples of one launch lie.  The host runs a tick as rounds of at most `sub`
// samples per stream (<= 6 hops, so no stream completes more than 8 frames per launch); round r starts at round_off = r * sub.
struct RaggedIn {
    const long long* offsets;  // [n + 1]: item i's chunk is pcm[offsets[i] .. offsets[i + 1]); null: pcm[i * chunk .. (i + 1) * chunk)
    long long max_len;         // chunk lengths are clamped to [0, max_len]
    long long round_off;
    int chunk;                 // uniform chunk length (offsets null)
    int sub;
};

// Item i's part of this launch: pcm[src .. src + len).  Offsets are clamped so that nothing outside
// [pcm + offsets[0], pcm + offsets[n]) is ever read, whatever the caller passed.
__device__ __forceinline__ void ragged_chunk(const RaggedIn& r, int i, int n, long long& src, int& len) {
    long long b, L;
    if (r.offsets) {
        const long long lo = __ldg(r.offsets), hi = max(lo, __ldg(r.offsets + n));
        b = min(max(__ldg(r.offsets + i), lo), hi);
        const long long e = min(max(__ldg(r.offsets + i + 1), b), hi);
        L = min(e - b, r.max_len);
    } else {
        b = (long long)i * r.chunk;
        L = r.chunk;
    }
    L = min(max(L - r.round_off, 0ll), (long long)r.sub);
    src = b + r.round_off;
    len = (int)L;
}

struct K1StreamSmem {
    K1Smem k1;
    // frame work list for this tile
    short fr_stream[K1_STREAMS_PER_CTA * 8];     // local stream slot
    short fr_sub[K1_STREAMS_PER_CTA * 8];        // j-th new frame of that stream
    int n_frames_tile;
    int st_id[K1_STREAMS_PER_CTA];
    int st_cnt[K1_STREAMS_PER_CTA];
    long long st_n0[K1_STREAMS_PER_CTA];
    long long st_ts0[K1_STREAMS_PER_CTA];
    long long st_c0[K1_STREAMS_PER_CTA];
    long long st_src[K1_STREAMS_PER_CTA];        // RAGGED: first sample of the stream's part of this launch, in pcm
    int st_len[K1_STREAMS_PER_CTA];              // RAGGED: its length
};

// One tick: stream ids[i] (or i) receives pcm[i * pcm_stride + 0 .. chunk).  A stream completes at most 8 frames per launch: the
// host feeds longer chunks as consecutive sub-chunks of the same rows (pcm_stride = the full chunk length), which the state machine
// cannot tell from separate ticks (Listener.update_vectors is chunking-independent).
// RAGGED: stream ids[i] receives its own part of the launch instead, pcm[src .. src + len) from ragged_chunk(rg, i) (chunk and
// pcm_stride are unused); any alignment, so only with PAIRS = false.
template <bool PAIRS, bool RAGGED = false>
__global__ void __launch_bounds__(K1_THREADS, 4)
mfcc_stream_kernel(const int16_t* __restrict__ pcm, const int* __restrict__ ids, int n, int chunk, int pcm_stride,
                   int hop, int used, float scale, MelTables tab, StreamState st, RaggedIn rg) {
    static_assert(!(PAIRS && RAGGED), "ragged chunks have any alignment");
    extern __shared__ __align__(16) unsigned char smem_raw[];
    K1StreamSmem& sm = *reinterpret_cast<K1StreamSmem*>(smem_raw);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, l16 = lane & 15, half = lane >> 4;
    FftLaneConst lc;
    load_lane_const(lc, tab.tw_stage, tab.tw_post, l16);
    float2* xch = sm.k1.xch + (warp * 2 + half) * XCH_ELEMS;
    load_tables(sm.k1.tab, tab, reinterpret_cast<float*>(smem_raw + sizeof(K1StreamSmem)));
    const bool big = tab.n_fft > 512;                           // see mfcc_batch_kernel
    unsigned char* big_base = smem_raw + ((sizeof(K1StreamSmem) + (size_t)tab.n_out * tab.n_filt * sizeof(float) + 15) & ~(size_t)15);
    float* const power = big ? reinterpret_cast<float*>(big_base) : sm.k1.power;
    const int ps = big ? K1_PSTRIDE_BIG : K1_PSTRIDE;
    float2* const xany = big ? reinterpret_cast<float2*>(big_base + (size_t)K1_TILE * K1_PSTRIDE_BIG * sizeof(float)) + warp * 1024 : sm.k1.xch + warp * 2 * XCH_ELEMS;
    const int n_tiles = (n + K1_STREAMS_PER_CTA - 1) / K1_STREAMS_PER_CTA;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int base = tile * K1_STREAMS_PER_CTA;
        // ---- bookkeeping: warp 0, one lane per stream; frame list by warp prefix sum
        if (warp == 0) {
            const int i = base + lane;
            int cnt = 0, sid = -1;
            long long n0 = 0, c0 = 0, ts0 = 0;
            if (i < n) {
                sid = ids ? ids[i] : i;
                n0 = st.n_samples[sid];
                c0 = frames_ready(n0, used, hop);
                int len = chunk;
                if (RAGGED) {
                    long long src;
                    ragged_chunk(rg, i, n, src, len);
                    sm.st_src[lane] = src; sm.st_len[lane] = len;
                }
                cnt = (int)(frames_ready(n0 + len, used, hop) - c0);
                ts0 = c0 * hop < n0 ? c0 * hop : n0;        // first absolute sample held in the tail
            }
            sm.st_id[lane] = sid; sm.st_n0[lane] = n0; sm.st_ts0[lane] = ts0; sm.st_cnt[lane] = cnt; sm.st_c0[lane] = c0;
            int incl = cnt;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { int v = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += v; }
            const int off = incl - cnt;
            for (int j = 0; j < cnt; ++j) { sm.fr_stream[off + j] = (short)lane; sm.fr_sub[off + j] = (short)j; }
            if (lane == 31) sm.n_frames_tile = incl;
        }
        __syncthreads();
        const int nf = sm.n_frames_tile;
        for (int r0 = 0; r0 < nf; r0 += K1_TILE) {
            const int nr = min(K1_TILE, nf - r0);
            // ---- phase A
            if (tab.n_fft != 512) {
#pragma unroll 1
                for (int slot = warp; slot < nr; slot += K1_WARPS) {               // generic n_fft: one frame per warp at a time
                    const int t = sm.fr_stream[r0 + slot];
                    const long long a0 = (sm.st_c0[t] + sm.fr_sub[r0 + slot]) * hop, n0 = sm.st_n0[t];
                    const int16_t* chunk_p = pcm + (RAGGED ? sm.st_src[t] : (long long)(base + t) * pcm_stride);
                    FrameSrc<int16_t> src;
                    src.used = used;
                    if (a0 >= n0) { src.len0 = 0; src.p0 = chunk_p; src.p1 = chunk_p + (a0 - n0); }
                    else {
                        src.len0 = (int)min((long long)used, n0 - a0);
                        src.p0 = st.tail + (long long)sm.st_id[t] * st.tail_cap + (a0 - sm.st_ts0[t]);
                        src.p1 = chunk_p;
                    }
                    fft_any_power<int16_t>(src, tab.n_fft, tab.tw_any, xany, power + slot * ps, scale, lane);
                }
            } else
#pragma unroll 1
            for (int pass = 0; pass * (K1_WARPS * 2) < nr; ++pass) {
                const int slot = pass * (K1_WARPS * 2) + warp * 2 + half;
                const bool active = slot < nr;
                cpx z[16];
                if (active) {
                    const int t = sm.fr_stream[r0 + slot];
                    const long long a0 = (sm.st_c0[t] + sm.fr_sub[r0 + slot]) * hop;     // absolute first sample
                    const long long n0 = sm.st_n0[t];
                    const int16_t* chunk_p = pcm + (RAGGED ? sm.st_src[t] : (long long)(base + t) * pcm_stride);
                    FrameSrc<int16_t> src;
                    src.used = used;
                    if (a0 >= n0) { src.len0 = 0; src.p0 = chunk_p; src.p1 = chunk_p + (a0 - n0); }
                    else {
                        src.len0 = (int)min((long long)used, n0 - a0);
                        src.p0 = st.tail + (long long)sm.st_id[t] * st.tail_cap + (a0 - sm.st_ts0[t]);
                        src.p1 = chunk_p;
                    }
#pragma unroll
                    for (int n1 = 0; n1 < 16; ++n1) z[n1] = load_elem<int16_t, PAIRS>(src, 16 * n1 + l16);
                } else {
#pragma unroll
                    for (int n1 = 0; n1 < 16; ++n1) z[n1] = {0.f, 0.f};
                }
                fft512_power(z, lc, xch, sm.k1.power + slot * K1_PSTRIDE, scale, l16, active);
            }
            __syncthreads();
            // ---- phase B: rows go straight into the ring (rows are 16-byte aligned and padded)
            if (threadIdx.x < nr) {
                const int t = sm.fr_stream[r0 + threadIdx.x];
                const long long k = sm.st_c0[t] + sm.fr_sub[r0 + threadIdx.x];
                float* row = st.ring + ((long long)sm.st_id[t] * st.ring_rows + (int)(k % st.ring_rows)) * st.row_stride;
                mel_log_dct<true>(power + threadIdx.x * ps, sm.k1.tab, tab, row);
            }
            __syncthreads();
        }
        // ---- tail + counter update: one warp per stream, all reads of the old tail precede the writes
        for (int t = warp; t < K1_STREAMS_PER_CTA; t += K1_WARPS) {
            const int sid = sm.st_id[t];
            if (sid < 0) continue;
            const long long n0 = sm.st_n0[t], n1 = n0 + (RAGGED ? sm.st_len[t] : chunk), ts0 = sm.st_ts0[t];
            const long long c1 = sm.st_c0[t] + sm.st_cnt[t];
            const long long ts1 = c1 * hop < n1 ? c1 * hop : n1;
            const int len1 = (int)(n1 - ts1);
            const int n_old = ts1 < n0 ? (int)(n0 - ts1) : 0;       // part that comes from the old tail
            int16_t* tl = st.tail + (long long)sid * st.tail_cap;
            const int16_t* chunk_p = pcm + (RAGGED ? sm.st_src[t] : (long long)(base + t) * pcm_stride);
            if (n_old > 0) {
                int16_t keep[64];                                    // tail_cap <= 2048 = 64 * 32
                const int off = (int)(ts1 - ts0);
#pragma unroll 1
                for (int j = 0; j * 32 < n_old; ++j) { int i = j * 32 + lane; keep[j & 63] = i < n_old ? tl[off + i] : (int16_t)0; }
                __syncwarp();
#pragma unroll 1
                for (int j = 0; j * 32 < n_old; ++j) { int i = j * 32 + lane; if (i < n_old) tl[i] = keep[j & 63]; }
            }
            const int16_t* srcp = chunk_p + (ts1 > n0 ? ts1 - n0 : 0);
            int16_t* dstp = tl + n_old;
            const int m = len1 - n_old;                              // samples copied from the chunk
            int done = 0;
            if ((((uintptr_t)srcp | (uintptr_t)dstp) & 15) == 0) {   // 16-byte vectors (default geometry)
                const int nv = m >> 3;
                for (int v = lane; v < nv; v += 32)
                    reinterpret_cast<int4*>(dstp)[v] = __ldg(reinterpret_cast<const int4*>(srcp) + v);
                done = nv << 3;
            }
            for (int i = done + lane; i < m; i += 32) dstp[i] = srcp[i];
            if (lane == 0) st.n_samples[sid] = n1;
        }
        __syncthreads();
    }
}

}  // namespace pb
