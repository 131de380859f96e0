// corpus.cuh -- recorded corpora (pb_score_corpus): a batch of whole recordings scored on the device in one call, the hot
// path of precise-simulate (precise/scripts/simulate.py:92-129) and of false-activation mining
// (precise/scripts/train_incremental.py:113-137).
//
// Frame buffer.  Row 0 is zero; then each recording r brings n_features - 1 zero rows followed by its nf_r MFCC frames, rows
// of row_stride floats (the MFCC width rounded up to 4, as the ring).  A window is n_features contiguous rows starting at its
// row of the window table, so the network kernels read it in place (K2In's predict mode) and no window is materialised.
// A window before the recording's first frame starts in the zero prefix; one with no frame at all starts at row 0, whose
// n_features rows are all zero (row 0 and recording 0's prefix -- every later prefix follows a frame).
//
// K1 runs over frame PAIRS, frames 2q and 2q + 1 of one recording: the fast kernel gives the frame of local parity h to
// half-warp h, as mfcc_fast_batch_kernel gives frame g to half g & 1, so each frame takes exactly the arithmetic it takes in
// pb_mfcc of its recording alone.  The generic kernel's per-frame code does not depend on where a frame sits.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "gru_kernels.cuh"
#include "mfcc_fast.cuh"
#include "mfcc_kernels.cuh"

namespace pb {

enum { CORPUS_LISTENER = 0, CORPUS_SIMULATE = 1 };

// Frames row .. row + n - 1 (n = 1 or 2) of the frame buffer, from samples src + k hop of the packed PCM.
struct CorpusPair {
    long long src;
    long long row;
    int n;
    int pad;
};

// One recording as K1's plan sees it, in the order of its pair list (fast recordings first, then generic ones).
struct CorpusRec {
    long long src;                   // first sample in the packed PCM
    long long row;                   // frame-buffer row of frame 0
    long long nf;                    // frames
    long long pair0;                 // first pair in the list; the entry after the last recording holds the total
};

// Largest j in [0, n) with a[j] <= v (a non-decreasing, a[0] <= v).
__device__ __forceinline__ int corpus_find(const long long* a, int n, long long v) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(a + mid) <= v) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// One thread per pair: pair p of the list.
__global__ void __launch_bounds__(256) corpus_pairs_kernel(const CorpusRec* __restrict__ recs, int n_rec, long long n_pairs,
                                                           int hop, CorpusPair* __restrict__ pairs) {
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_pairs) return;
    const long long* pair0 = &recs[0].pair0;
    int lo = 0, hi = n_rec - 1;                                   // corpus_find over the strided pair0 fields
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(pair0 + 4 * mid) <= p) lo = mid; else hi = mid - 1;
    }
    const CorpusRec r = recs[lo];
    const long long q = p - r.pair0;
    CorpusPair e;
    e.src = r.src + 2 * q * hop;
    e.row = r.row + 2 * q;
    e.n = r.nf - 2 * q >= 2 ? 2 : 1;
    e.pad = 0;
    pairs[p] = e;
}

// One thread per window: its start row.  win0 [n_rec + 1] = the windows' prefix, frow [n_rec] = row of each recording's
// frame 0.  LISTENER: window k is Listener.update's after (k + 1) chunk samples, the 29 rows ending at the last released
// frame.  SIMULATE: window k holds frames k hops .. k hops + T - 1 (simulate.py:96-99).
__global__ void __launch_bounds__(256) corpus_windows_kernel(const long long* __restrict__ win0, const long long* __restrict__ frow,
                                                             int n_rec, long long n_win, int schedule, long long chunk,
                                                             int rel_window, int hop, int T, long long* __restrict__ starts) {
    const long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= n_win) return;
    const int r = corpus_find(win0, n_rec, w);
    const long long k = w - __ldg(win0 + r), fr = __ldg(frow + r);
    long long s;
    if (schedule == CORPUS_SIMULATE) {
        s = fr + k * (chunk / hop);
    } else {
        const long long N = (k + 1) * chunk;
        const long long rel = N >= rel_window ? (N - rel_window) / hop + 1 : 0;
        s = rel == 0 ? 0 : fr + rel - T;
    }
    starts[w] = s;
}

// ------------------------------------------------------------------------------------------------
// K1, aligned geometry: mfcc_fast_batch_kernel's loop over a pair list.  Every pair's samples start 16-byte aligned.
__global__ void __launch_bounds__(K1F_THREADS, 4)
mfcc_fast_corpus_kernel(const int16_t* __restrict__ pcm, const CorpusPair* __restrict__ pairs, long long n_pairs, int hop,
                        float scale, MelTables tab, FastTables ft, float* __restrict__ rows, int row_stride) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    K1FWarp* wsm = reinterpret_cast<K1FWarp*>(smem_raw);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, l16 = lane & 15, half = lane >> 4;
    K1FWarp& ws = wsm[warp];
    const K1FTab tb = load_fast_tables(smem_raw + K1F_WARPS * sizeof(K1FWarp), tab, ft);
    if (lane == 0) { mbar_init(&ws.bar[0], 1); mbar_init(&ws.bar[1], 1); fence_mbar_init(); }
    if (l16 == 0) ws.part[half][128] = 0.f;
    int eoff[8];
    {
        const int rot = ((l16 >> 2) + (half << 2)) & 7;
#pragma unroll
        for (int i = 0; i < 8; ++i) eoff[i] = ((i + rot) & 7) * 16 + l16;
    }
    FftLaneConst lc;
    load_lane_const(lc, tab.tw_stage, tab.tw_post, l16);
    __syncthreads();

    const long long gwarp = (long long)blockIdx.x * K1F_WARPS + warp, nwarps = (long long)gridDim.x * K1F_WARPS;
    auto issue = [&](const CorpusPair& e, int stage) {          // lane 0: bulk copies for the pair's frames
        fence_proxy_async();
        mbar_expect_tx(&ws.bar[stage], 1024u * e.n);
        for (int hf = 0; hf < e.n; ++hf) bulk_g2s(ws.buf[stage][hf], pcm + e.src + (long long)hf * hop, 1024u, &ws.bar[stage]);
    };
    long long pair = gwarp;
    int it = 0;
    CorpusPair cur{};
    if (pair < n_pairs) {
        cur = pairs[pair];
        if (lane == 0) issue(cur, 0);
    }
    for (; pair < n_pairs; pair += nwarps, ++it) {
        const int stage = it & 1;
        const long long next = pair + nwarps;
        CorpusPair nx{};
        if (next < n_pairs) {
            nx = pairs[next];
            if (lane == 0) issue(nx, stage ^ 1);
        }
        const bool active = half < cur.n;
        fast_pass(ws, stage, (uint32_t)((it >> 1) & 1), lc, tb, ft, tab, scale, eoff, l16, half, active,
                  rows + (cur.row + (active ? half : 0)) * row_stride);
        cur = nx;
    }
}

// K1, any geometry and alignment: mfcc_batch_kernel's per-frame code over a pair list, 16 pairs (32 frame slots) per tile.
__global__ void __launch_bounds__(K1_THREADS, 4)
mfcc_corpus_kernel(const int16_t* __restrict__ pcm, const CorpusPair* __restrict__ pairs, long long n_pairs, int hop, int used,
                   float scale, MelTables tab, float* __restrict__ rows, int row_stride) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    K1Smem& sm = *reinterpret_cast<K1Smem*>(smem_raw);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, l16 = lane & 15, half = lane >> 4;
    FftLaneConst lc;
    load_lane_const(lc, tab.tw_stage, tab.tw_post, l16);
    float2* xch = sm.xch + (warp * 2 + half) * XCH_ELEMS;
    load_tables(sm.tab, tab, reinterpret_cast<float*>(smem_raw + sizeof(K1Smem)));
    const bool big = tab.n_fft > 512;
    unsigned char* big_base = smem_raw + ((sizeof(K1Smem) + (size_t)tab.n_out * tab.n_filt * sizeof(float) + 15) & ~(size_t)15);
    float* const power = big ? reinterpret_cast<float*>(big_base) : sm.power;
    const int ps = big ? K1_PSTRIDE_BIG : K1_PSTRIDE;
    float2* const xany = big ? reinterpret_cast<float2*>(big_base + (size_t)K1_TILE * K1_PSTRIDE_BIG * sizeof(float)) + warp * 1024 : sm.xch + warp * 2 * XCH_ELEMS;
    __syncthreads();
    // slot s of a tile: frame s & 1 of pair tile * 16 + s / 2; src < 0 marks an empty slot
    auto frame = [&](long long tile, int slot, long long& src, long long& row) {
        const long long p = tile * (K1_TILE / 2) + (slot >> 1);
        src = -1;
        if (p >= n_pairs) return;
        const CorpusPair e = pairs[p];
        if ((slot & 1) >= e.n) return;
        src = e.src + (long long)(slot & 1) * hop;
        row = e.row + (slot & 1);
    };
    const long long n_tiles = (n_pairs + K1_TILE / 2 - 1) / (K1_TILE / 2);
    for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        if (tab.n_fft != 512) {
#pragma unroll 1
            for (int slot = warp; slot < K1_TILE; slot += K1_WARPS) {
                long long src, row;
                frame(tile, slot, src, row);
                if (src < 0) continue;
                FrameSrc<int16_t> fs;
                fs.p0 = pcm + src; fs.p1 = fs.p0; fs.len0 = used; fs.used = used;
                fft_any_power<int16_t>(fs, tab.n_fft, tab.tw_any, xany, power + slot * ps, scale, lane);
            }
        } else
#pragma unroll 1
        for (int pass = 0; pass < K1_TILE / (K1_WARPS * 2); ++pass) {
            const int slot = pass * (K1_WARPS * 2) + warp * 2 + half;
            long long src, row;
            frame(tile, slot, src, row);
            const bool active = src >= 0;
            cpx z[16];
            if (active) {
                FrameSrc<int16_t> fs;
                fs.p0 = pcm + src; fs.p1 = fs.p0; fs.len0 = used; fs.used = used;
#pragma unroll
                for (int n1 = 0; n1 < 16; ++n1) z[n1] = load_elem<int16_t, false>(fs, 16 * n1 + l16);
            } else {
#pragma unroll
                for (int n1 = 0; n1 < 16; ++n1) z[n1] = {0.f, 0.f};
            }
            fft512_power(z, lc, xch, sm.power + slot * K1_PSTRIDE, scale, l16, active);
        }
        __syncthreads();
        if (threadIdx.x < K1_TILE) {
            long long src, row;
            frame(tile, threadIdx.x, src, row);
            if (src >= 0) mel_log_dct<false>(power + threadIdx.x * ps, sm.tab, tab, rows + row * row_stride);
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------
// Per-recording TriggerDetector (runner/precise_runner/runner.py:127-142) over the windows of each (model, recording).
struct CorpusTrig {
    const float* raw;                // [M][W]
    const double* conf;              // [M][W] or null: decoded here (listener)
    uint8_t* fired;                  // [M][W] or null
    int64_t* activations;            // [M][n_rec] or null
    int64_t* above;                  // [M][n_rec] or null (simulate)
    double* sum;                     // [M][n_rec] or null (simulate)
    const long long* win0;           // [n_rec + 1]
    long long W;
    int n_rec;
    int schedule;
    float hot_f, above_f;            // simulate: (float)(1 - threshold), (float)threshold
    int sim_reset;                   // simulate: -(8 * 2048) // chunk
};

// Listener: the decoder and detector (hot_threshold, trigger_level, trigger_reset) of row m over recording r, here row m's
// bank model.  The model pool's rows read theirs from their slot records (corpus_pool.cuh, CorpusPoolDP), and pairs, whose
// one row holds a model per "recording", from the slot record of recording r's model (corpus_pairs.cuh, CorpusPairsDP).
struct CorpusBankDP {
    DecodeParams dp[PB_MAX_MODELS];
    __device__ __forceinline__ const DecodeParams& operator()(int m, long long) const { return dp[m]; }
};

constexpr int CORPUS_TRIG_THREADS = 256;

// A warp per (row = blockIdx.y, recording).  Lanes load 32 consecutive windows at once (the next 32 are in flight while
// these are used) and decide hot in parallel; the detector's serial recurrence then runs over the warp's ballot of hot
// flags, identically in every lane, and lane j keeps fired of its window.
template <class DP>
__global__ void __launch_bounds__(CORPUS_TRIG_THREADS) corpus_trigger_kernel(const __grid_constant__ CorpusTrig P,
                                                                             const __grid_constant__ DP dps) {
    const int m = blockIdx.y, lane = threadIdx.x & 31;
    const long long r = (long long)blockIdx.x * (CORPUS_TRIG_THREADS / 32) + (threadIdx.x >> 5);
    if (r >= P.n_rec) return;                                     // whole warp
    const DecodeParams& d = dps(m, r);
    const bool sim = P.schedule == CORPUS_SIMULATE;
    const int level = sim ? 0 : d.trigger_level, reset = sim ? P.sim_reset : d.trigger_reset;
    const long long w0 = __ldg(P.win0 + r), w1 = __ldg(P.win0 + r + 1), off = (long long)m * P.W;
    const float* raw = P.raw + off;
    const double* conf = (!sim && P.conf) ? P.conf + off : nullptr;
    float v = w0 + lane < w1 ? __ldg(raw + w0 + lane) : 0.f;
    double c = conf && w0 + lane < w1 ? __ldg(conf + w0 + lane) : 0.0;
    int a = 0;
    long long acts = 0, above = 0;
    double sum = 0.0;
    for (long long b = w0; b < w1; b += 32) {
        const long long w = b + lane;
        const bool ok = w < w1;
        const bool more = w + 32 < w1;
        const float vn = more ? __ldg(raw + w + 32) : 0.f;
        const double cn = conf && more ? __ldg(conf + w + 32) : 0.0;
        bool hot;
        if (sim) {
            hot = v > P.hot_f;                                     // float32 comparisons, as numpy compares float32 outputs
            if (ok) { above += v > P.above_f; sum += (double)v; }
        } else {
            hot = (conf ? c : decode_one(v, d)) > d.hot_threshold;
        }
        const unsigned hm = __ballot_sync(0xffffffffu, ok && hot);
        const int cnt = (int)(w1 - b < 32 ? w1 - b : 32);
        unsigned fm = 0;
        for (int j = 0; j < cnt; ++j) {
            const bool h = hm >> j & 1u;
            if (h || a < 0) {
                a += 1;
                const bool f = a > level;
                if (f || (h && a < 0)) a = reset;
                if (f) fm |= 1u << j;
            } else if (a > 0) {
                a -= 1;
            }
        }
        if (ok && P.fired) P.fired[off + w] = (uint8_t)(fm >> lane & 1u);
        acts += __popc(fm);
        v = vn; c = cn;
    }
#pragma unroll
    for (int s = 16; s >= 1; s >>= 1) {
        above += __shfl_xor_sync(0xffffffffu, above, s);
        sum += __shfl_xor_sync(0xffffffffu, sum, s);
    }
    if (lane == 0) {
        const long long o = (long long)m * P.n_rec + r;
        if (P.activations) P.activations[o] = acts;
        if (P.above) P.above[o] = above;
        if (P.sum) P.sum[o] = sum;
    }
}

}  // namespace pb
