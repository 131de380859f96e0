// dataset.cuh -- pool models over labelled clips (pb_score_dataset): one network input per clip, vectorize's
// (precise/vectorization.py:62-84), and per-model statistics over the outputs: what precise-test (stats.py), precise-graph
// (scripts/graph.py:147-152) and precise-calc-threshold (scripts/calc_threshold.py:66-83) compute from
// Runner.predict(vectorize(clip)).
//
// K1 and the scans are the corpus calls' (corpus.cuh, corpus_pool.cuh, corpus_pairs.cuh) over a frame buffer whose recordings
// are the cropped clips, one window each.  New here:
//   dataset_stats_kernel  one thread per scored entry.  The float32 thresholds sit in shared memory and an entry's histogram
//                         bin is a binary search over them.  Every statistic is an int64 sum, so the result does not depend
//                         on the order of the atomics and adds across calls.
//     cross product (PAIRS = false): blockIdx.y is the statistics row, so a CTA owns one row: its histogram is built in shared
//                         memory and flushed with one atomicAdd per non-zero bin, and the counts and fit sums are kept per
//                         thread over the CTA's DS_ITERS entries, then reduced per warp to one atomic per sum and label.
//     pairs (PAIRS = true): an entry's row comes from its pair.  Lanes with the same (row, label) are found with
//                         __match_any_sync, as pool_route_kernel finds the lanes of one model, and reduced before the atomics;
//                         lanes with the same histogram bin likewise.
//   Misclassified entries are compacted as pairs_hits_kernel compacts hits: a warp ballot and one atomicAdd per warp.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pb {

constexpr int DS_THREADS = 256;
constexpr int DS_ITERS = 16;               // entries per thread of the cross product's CTA
constexpr int DS_MAX_THR = 1024;

struct DatasetStats {
    const float* raw;                // cross product: [rows of the launch][n]; pairs: [n]
    const uint8_t* targets;          // [n_rec]: != 0 = wake word
    const int2* pairs;               // pairs: [n] (statistics row, recording)
    const float* thr;                // [n_thr] strictly ascending, or null (no histogram)
    int n_thr;
    int row0;                        // cross product: statistics row of blockIdx.y == 0
    long long n;                     // cross product: recordings; pairs: entries of the batch
    long long base;                  // pairs: index of the batch's entry 0 in the miss list
    int64_t* count;                  // [k][2] or null
    int64_t* hist;                   // [k][2][2 n_thr + 1] or null
    int64_t* fit;                    // [k][2][3] or null
    float miss_thr;
    int64_t* miss;                   // [capacity] or null (capacity 0)
    long long capacity;
    unsigned long long* n_miss;      // null: no miss list
};

// Histogram bin of x: 2 j + 1 when x == t_j, else 2 j for t_(j-1) < x < t_j (t_(-1) = -inf, t_n = +inf).  NaN: bin 0.
__device__ __forceinline__ int dataset_bin(const float* t, int n, float x) {
    int lo = 0, hi = n;                                               // lo = #(t_j < x)
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (t[mid] < x) lo = mid + 1; else hi = mid;
    }
    return 2 * lo + (lo < n && t[lo] == x);
}

// calc_threshold.py:66-70 for one output: v = -log(1 / x - 1), the 1 / x - 1 in float32 as decode_one has it.  False for the
// outputs calc_threshold drops (0 and 1) and for those without a finite v (NaN, and float32 denormals, whose reciprocal is inf).
__device__ __forceinline__ bool dataset_fit(float x, long long& s1, long long& s2) {
    if (x == 0.0f || x == 1.0f) return false;
    const double v = -log((double)__fsub_rn(__fdiv_rn(1.0f, x), 1.0f));
    if (!isfinite(v)) return false;
    s1 = llrint(v * 4294967296.0);
    s2 = llrint(v * v * 16777216.0);
    return true;
}

__device__ __forceinline__ long long warp_sum(long long v) {
#pragma unroll
    for (int s = 16; s >= 1; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
    return v;
}

__device__ __forceinline__ void dataset_add(int64_t* p, long long v) {
    if (v) atomicAdd(reinterpret_cast<unsigned long long*>(p), (unsigned long long)v);
}

// Whole warp: entry `index` of the lanes with `miss` set goes to the list.
__device__ __forceinline__ void dataset_miss(const DatasetStats& D, bool miss, long long index, int lane) {
    const unsigned b = __ballot_sync(0xffffffffu, miss);
    if (b == 0) return;
    unsigned long long at = 0;
    if (lane == 0) at = atomicAdd(D.n_miss, (unsigned long long)__popc(b));
    at = __shfl_sync(0xffffffffu, at, 0);
    const unsigned long long pos = at + (unsigned)__popc(b & ((1u << lane) - 1u));
    if (miss && pos < (unsigned long long)D.capacity) D.miss[pos] = index;
}

template <bool PAIRS>
__global__ void __launch_bounds__(DS_THREADS) dataset_stats_kernel(const __grid_constant__ DatasetStats D) {
    __shared__ float s_thr[DS_MAX_THR];
    __shared__ unsigned s_hist[PAIRS ? 1 : 2 * (2 * DS_MAX_THR + 1)];
    const int lane = threadIdx.x & 31, bins = 2 * D.n_thr + 1;
    const bool hist = D.hist != nullptr;
    if (hist) {
        for (int i = threadIdx.x; i < D.n_thr; i += DS_THREADS) s_thr[i] = __ldg(D.thr + i);
        if (!PAIRS)
            for (int i = threadIdx.x; i < 2 * bins; i += DS_THREADS) s_hist[i] = 0;
        __syncthreads();
    }
    if (PAIRS) {
        const long long q = (long long)blockIdx.x * DS_THREADS + threadIdx.x;
        const bool ok = q < D.n;
        int key = -1;                                                 // 2 row + label
        float x = 0.f;
        if (ok) {
            const int2 e = __ldg(D.pairs + q);
            key = 2 * e.x + (__ldg(D.targets + e.y) != 0);
            x = __ldg(D.raw + q);
        }
        if (D.n_miss) dataset_miss(D, ok && (x > D.miss_thr) != (bool)(key & 1), q + D.base, lane);
        if (hist) {
            const long long hk = ok ? (long long)key * bins + dataset_bin(s_thr, D.n_thr, x) : -1;
            const unsigned peers = __match_any_sync(0xffffffffu, hk);
            if (ok && lane == __ffs(peers) - 1) dataset_add(D.hist + hk, __popc(peers));
        }
        if (D.count || D.fit) {
            long long s1 = 0, s2 = 0;
            const bool f = ok && D.fit && dataset_fit(x, s1, s2);
            if (!f) s1 = s2 = 0;
            const unsigned peers = __match_any_sync(0xffffffffu, key);
            unsigned rem = __ballot_sync(0xffffffffu, ok);
            while (rem) {                                             // one round per (row, label) of the warp
                const int leader = __ffs(rem) - 1;
                const unsigned grp = __shfl_sync(0xffffffffu, peers, leader);
                const bool mine = grp >> lane & 1u;
                const long long c = __popc(grp), nf = __popc(__ballot_sync(0xffffffffu, mine && f));
                const long long a1 = warp_sum(mine ? s1 : 0), a2 = warp_sum(mine ? s2 : 0);
                if (lane == leader) {
                    if (D.count) dataset_add(D.count + key, c);
                    if (D.fit) {
                        dataset_add(D.fit + 3 * key, nf);
                        dataset_add(D.fit + 3 * key + 1, a1);
                        dataset_add(D.fit + 3 * key + 2, a2);
                    }
                }
                rem &= ~grp;
            }
        }
    } else {
        const int row = D.row0 + blockIdx.y;
        const float* raw = D.raw + (long long)blockIdx.y * D.n;
        long long cnt[2] = {0, 0}, nf[2] = {0, 0}, s1[2] = {0, 0}, s2[2] = {0, 0};
#pragma unroll 1
        for (int it = 0; it < DS_ITERS; ++it) {
            const long long r = ((long long)blockIdx.x * DS_ITERS + it) * DS_THREADS + threadIdx.x;
            if (r - threadIdx.x >= D.n) break;                        // whole CTA
            const bool ok = r < D.n;
            const float x = ok ? __ldg(raw + r) : 0.f;
            const int label = ok ? __ldg(D.targets + r) != 0 : 0;
            if (D.n_miss) dataset_miss(D, ok && (x > D.miss_thr) != (bool)label, (long long)row * D.n + r, lane);
            if (!ok) continue;
            if (hist) atomicAdd(&s_hist[label * bins + dataset_bin(s_thr, D.n_thr, x)], 1u);
            long long a1 = 0, a2 = 0;
            const bool f = D.fit && dataset_fit(x, a1, a2);
#pragma unroll
            for (int l = 0; l < 2; ++l) {                             // predicated, so that the sums stay in registers
                const bool m = label == l;
                cnt[l] += m;
                nf[l] += m && f;
                s1[l] += m && f ? a1 : 0;
                s2[l] += m && f ? a2 : 0;
            }
        }
#pragma unroll
        for (int l = 0; l < 2; ++l) {
            const long long c = warp_sum(cnt[l]);
            if (D.fit) {
                const long long f = warp_sum(nf[l]), a1 = warp_sum(s1[l]), a2 = warp_sum(s2[l]);
                if (lane == 0) {
                    int64_t* o = D.fit + 3 * (2 * row + l);
                    dataset_add(o, f);
                    dataset_add(o + 1, a1);
                    dataset_add(o + 2, a2);
                }
            }
            if (lane == 0 && D.count) dataset_add(D.count + 2 * row + l, c);
        }
        if (hist) {
            __syncthreads();
            for (int i = threadIdx.x; i < 2 * bins; i += DS_THREADS)
                dataset_add(D.hist + (long long)row * 2 * bins + i, s_hist[i]);
        }
    }
}

}  // namespace pb
