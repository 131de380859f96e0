// history.cuh -- stream audio history (pb_set_history, pb_set_stream_history, pb_read_history).
//
// A pool of rows, each holding the last `cap` int16 samples of one stream (cap = history_samples rounded up to a multiple of
// 8).  Invariant: sample k of a stream's audio, counted as n_samples counts, lives at row position k mod cap.  A [max_streams]
// row map says which row a stream owns (-1 = off), and a [max_streams] history start says from which sample on the row holds
// this life of the stream: positions before it read as 0.
//
// history_append_kernel: one warp per tick item, launched before K1 on the tick's stream, so it reads the pre-tick n_samples.
// It takes the item's chunk exactly as K1 does (ragged_chunk with round offset 0 and sub = max_len), keeps its last cap
// samples and copies them in at most two pieces (before and after the wrap).  Each piece goes as 16-byte vectors when source
// and destination share their alignment mod 16 -- a uniform tick of a multiple-of-8 chunk on a handle that never went ragged
// -- with 2-byte accesses at its ends; otherwise as 2-byte accesses, consecutive lanes on consecutive samples.  Row writes
// use streaming stores (evict-first): only pb_read_history reads them again.
// history_read_kernel: one CTA per item, one thread per output sample, zero before the history start.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "mfcc_kernels.cuh"

namespace pb {

constexpr int HIST_THREADS = 256;

struct HistPool {
    int16_t* rows;                     // [max_rows][cap]
    int* row_of;                       // [max_streams] row of each stream, -1 = off
    long long* start;                  // [max_streams] history start (a sample count)
    int cap;                           // row length, a multiple of 8
};

// dst[0, len) = src[0, len) by the 32 lanes of a warp, as accesses of type V (src and dst share their alignment mod
// sizeof(V)): 2-byte accesses up to dst's first V boundary and after its last, U loads in flight per lane before the stores.
template <typename V, int U>
__device__ __forceinline__ void warp_copy_as(const int16_t* __restrict__ src, int16_t* __restrict__ dst, int len, int lane) {
    constexpr int E = (int)sizeof(V) / 2;                          // samples per access
    const int head = min(len, (int)(((sizeof(V) - ((uintptr_t)dst & (sizeof(V) - 1))) & (sizeof(V) - 1)) >> 1));
    if (lane < head) __stcs(dst + lane, src[lane]);
    const int nv = (len - head) / E;
    const V* s = reinterpret_cast<const V*>(src + head);
    V* d = reinterpret_cast<V*>(dst + head);
    for (int v0 = lane; v0 < nv; v0 += 32 * U) {
        V x[U];
#pragma unroll
        for (int u = 0; u < U; ++u)
            if (v0 + 32 * u < nv) x[u] = s[v0 + 32 * u];
#pragma unroll
        for (int u = 0; u < U; ++u)
            if (v0 + 32 * u < nv) __stcs(d + v0 + 32 * u, x[u]);
    }
    const int t0 = head + E * nv;
    if (lane < len - t0) __stcs(dst + t0 + lane, src[t0 + lane]);
}

// dst[0, len) = src[0, len): 16-byte accesses where source and destination share their alignment mod 16, else 4-byte ones
// where they share it mod 4, else 2-byte ones.
__device__ __forceinline__ void warp_copy_i16(const int16_t* __restrict__ src, int16_t* __restrict__ dst, int len, int lane) {
    const uintptr_t x = (uintptr_t)src ^ (uintptr_t)dst;
    if ((x & 15) == 0) warp_copy_as<uint4, 4>(src, dst, len, lane);
    else if ((x & 3) == 0) warp_copy_as<int, 8>(src, dst, len, lane);
    else warp_copy_as<short, 8>(src, dst, len, lane);
}

// Appends item i's chunk of a tick to the row of stream ids[i] (or i), if it has one.
__global__ void __launch_bounds__(HIST_THREADS)
history_append_kernel(const int16_t* __restrict__ pcm, RaggedIn rg, const int* __restrict__ ids, int n,
                      const long long* __restrict__ n_samples, HistPool P) {
    const int i = blockIdx.x * (HIST_THREADS / 32) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (i >= n) return;
    const int sid = ids ? ids[i] : i;
    const int row = P.row_of[sid];
    if (row < 0) return;
    long long src;
    int len;
    ragged_chunk(rg, i, n, src, len);
    long long k0 = n_samples[sid];
    if (len > P.cap) {                                             // only the last cap samples survive
        src += len - P.cap;
        k0 += len - P.cap;
        len = P.cap;
    }
    if (len <= 0) return;
    const int p0 = (int)(k0 % P.cap);
    int16_t* base = P.rows + (long long)row * P.cap;
    const int l1 = min(len, P.cap - p0);
    warp_copy_i16(pcm + src, base + p0, l1, lane);
    if (len > l1) warp_copy_i16(pcm + src + l1, base, len - l1, lane);
}

// out[i][j] = sample N - samples + j of stream ids[i] (or i), N its n_samples; 0 before its history start, and for a stream
// that is off or an id outside [0, max_streams).
__global__ void __launch_bounds__(HIST_THREADS)
history_read_kernel(HistPool P, const long long* __restrict__ n_samples, const int* __restrict__ ids, int max_streams,
                    int samples, int16_t* __restrict__ out) {
    const long long i = blockIdx.x;
    const int sid = ids ? ids[i] : (int)i;
    int16_t* o = out + i * samples;
    const int row = (sid >= 0 && sid < max_streams) ? P.row_of[sid] : -1;
    if (row < 0) {
        for (int j = threadIdx.x; j < samples; j += HIST_THREADS) o[j] = 0;
        return;
    }
    const long long k0 = n_samples[sid] - samples;                 // sample of out[i][0]
    const int zeros = (int)min((long long)samples, max(P.start[sid] - k0, 0ll));
    const int p = (int)(((k0 % P.cap) + P.cap) % P.cap);
    const int16_t* r = P.rows + (long long)row * P.cap;
    for (int j = threadIdx.x; j < samples; j += HIST_THREADS) {
        int q = p + j;                                             // j < samples <= cap
        if (q >= P.cap) q -= P.cap;
        o[j] = j < zeros ? (int16_t)0 : r[q];
    }
}

// Stream sids[j] gets row rows[j]: -1 switches it off, a row switches it on with its history starting at its n_samples.
__global__ void history_set_kernel(HistPool P, const long long* __restrict__ n_samples, const int* __restrict__ sids,
                                   const int* __restrict__ rows, long long k) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= k) return;
    const int sid = sids[j];
    P.row_of[sid] = rows[j];
    if (rows[j] >= 0) P.start[sid] = n_samples[sid];
}

// The history of streams ids[i] (or i) restarts at their n_samples (after pb_clear and pb_import_streams).
__global__ void history_restart_kernel(HistPool P, const long long* __restrict__ n_samples, const int* __restrict__ ids,
                                       long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int sid = ids ? ids[i] : (int)i;
    P.start[sid] = n_samples[sid];
}

}  // namespace pb
