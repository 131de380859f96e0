// stream_state.cuh -- stream state export / import (pb_export_streams, pb_import_streams).
//
// A record is one stream's listener state in the layout include/precise_b200.h documents: a 96 B pb_stream_state_header
// (format, the front-end fields that fix the layout, n_samples, each bank model's TriggerDetector.activation), then the tail
// and the MFCC ring copied whole, padding columns included.  Copying them whole keeps the record independent of how K1
// indexes them, and the bank kernel's 64 B row loads get back exactly the bits K1 left.
//
// export_state_kernel / import_state_kernel: one warp per record, 16-byte vectors; a record is one contiguous piece, so every
// access is coalesced whatever the order of the ids.  The record side uses streaming hints (evict-first): the kernels never
// read it again.  validate_state_kernel: one thread per record, reduced with a warp ballot and one atomic per warp and result.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/precise_b200.h"
#include "mfcc_kernels.cuh"

namespace pb {

constexpr int STATE_THREADS = 256;
constexpr int STATE_HEADER_VECS = (int)(sizeof(pb_stream_state_header) / 16);
constexpr int STATE_HEAD_WORDS = 12;       // magic, version, num_models and the 9 front-end fields: equal on export and import
constexpr int STATE_BAD_N_SAMPLES = STATE_HEAD_WORDS + 1;
static_assert(sizeof(pb_stream_state_header) == 96 && sizeof(pb_stream_state_header) % 16 == 0, "record header layout");
static_assert(offsetof(pb_stream_state_header, n_samples) == 48 && offsetof(pb_stream_state_header, activation) == 64,
              "record header layout");

// What a handle's records look like.
struct StateLayout {
    unsigned head[STATE_HEAD_WORDS];   // the header's first 12 words for this handle
    int* trig[PB_MAX_MODELS];          // each bank model's TriggerDetector.activation; null past the last model
    int tail_vecs, ring_vecs;          // 16-byte vectors per stream of tail and ring
    long long rec_vecs;                // ... of a record: STATE_HEADER_VECS + tail_vecs + ring_vecs
};

// validate_state_kernel's result.  first = (record index << 8) | reason of the first bad record (~0 when none); reason k + 1
// names header word k (1 magic, 2 version, 3 num_models, 4.. the front-end fields), STATE_BAD_N_SAMPLES a negative n_samples.
struct StateCheck {
    unsigned long long first;
    unsigned bad;                      // number of bad records
    unsigned unaligned;                // 1 if a good record's n_samples is not a multiple of 8
};

// Header word k (of 24) of stream sid's record.
__device__ __forceinline__ unsigned state_header_word(const StateLayout& L, const StreamState& st, int sid, int k) {
    if (k < STATE_HEAD_WORDS) return L.head[k];
    if (k < 14) {
        const unsigned long long ns = (unsigned long long)st.n_samples[sid];
        return k == 12 ? (unsigned)ns : (unsigned)(ns >> 32);
    }
    if (k < 16) return 0u;                                          // reserved
    const int* t = L.trig[k - 16];
    return t ? (unsigned)t[sid] : 0u;
}

__global__ void __launch_bounds__(STATE_THREADS)
export_state_kernel(const __grid_constant__ StateLayout L, StreamState st, const int* __restrict__ ids, long long n,
                    uint4* __restrict__ out) {
    const long long r = (long long)blockIdx.x * (STATE_THREADS / 32) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (r >= n) return;
    const int sid = ids ? ids[r] : (int)r;
    uint4* rec = out + r * L.rec_vecs;
    if (lane < STATE_HEADER_VECS) {
        uint4 v;
        v.x = state_header_word(L, st, sid, 4 * lane);
        v.y = state_header_word(L, st, sid, 4 * lane + 1);
        v.z = state_header_word(L, st, sid, 4 * lane + 2);
        v.w = state_header_word(L, st, sid, 4 * lane + 3);
        __stcs(rec + lane, v);
    }
    const uint4* tail = reinterpret_cast<const uint4*>(st.tail + (long long)sid * st.tail_cap);
    const uint4* ring = reinterpret_cast<const uint4*>(st.ring + (long long)sid * st.ring_rows * st.row_stride);
    const int nv = L.tail_vecs + L.ring_vecs;
    rec += STATE_HEADER_VECS;
    for (int v0 = lane; v0 < nv; v0 += 32 * 4) {                    // 4 loads in flight per lane before the first store
        uint4 x[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int v = v0 + 32 * u;
            if (v < nv) x[u] = v < L.tail_vecs ? tail[v] : ring[v - L.tail_vecs];
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int v = v0 + 32 * u;
            if (v < nv) __stcs(rec + v, x[u]);
        }
    }
}

// Writes validated records: n_samples, the activations of the handle's models, tail and ring.
__global__ void __launch_bounds__(STATE_THREADS)
import_state_kernel(const __grid_constant__ StateLayout L, StreamState st, const int* __restrict__ ids, long long n,
                    const uint4* __restrict__ in) {
    const long long r = (long long)blockIdx.x * (STATE_THREADS / 32) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (r >= n) return;
    const int sid = ids ? ids[r] : (int)r;
    const uint4* rec = in + r * L.rec_vecs;
    if (lane == 0) {
        const uint4 w = __ldcs(rec + 3);                            // words 12..15: n_samples, reserved
        st.n_samples[sid] = (long long)(((unsigned long long)w.y << 32) | w.x);
    } else if (lane <= PB_MAX_MODELS) {
        int* t = L.trig[lane - 1];
        if (t) t[sid] = __ldcs(reinterpret_cast<const int*>(rec) + 15 + lane);
    }
    uint4* tail = reinterpret_cast<uint4*>(st.tail + (long long)sid * st.tail_cap);
    uint4* ring = reinterpret_cast<uint4*>(st.ring + (long long)sid * st.ring_rows * st.row_stride);
    const int nv = L.tail_vecs + L.ring_vecs;
    rec += STATE_HEADER_VECS;
    for (int v0 = lane; v0 < nv; v0 += 32 * 4) {
        uint4 x[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int v = v0 + 32 * u;
            if (v < nv) x[u] = __ldcs(rec + v);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int v = v0 + 32 * u;
            if (v < nv) {
                if (v < L.tail_vecs) tail[v] = x[u];
                else ring[v - L.tail_vecs] = x[u];
            }
        }
    }
}

// One thread per record: the header words against this handle's, then n_samples >= 0; a good record whose n_samples is not a
// multiple of 8 sets `unaligned`.  out starts as {~0, 0, 0}.
__global__ void __launch_bounds__(STATE_THREADS)
validate_state_kernel(const __grid_constant__ StateLayout L, const uint4* __restrict__ in, long long n, StateCheck* out) {
    const long long r = (long long)blockIdx.x * STATE_THREADS + threadIdx.x;
    int reason = 0;
    bool odd = false;
    if (r < n) {
        const uint4* rec = in + r * L.rec_vecs;
        unsigned w[16];
#pragma unroll
        for (int v = 0; v < 4; ++v) {
            const uint4 x = __ldcs(rec + v);
            w[4 * v] = x.x; w[4 * v + 1] = x.y; w[4 * v + 2] = x.z; w[4 * v + 3] = x.w;
        }
#pragma unroll
        for (int k = STATE_HEAD_WORDS - 1; k >= 0; --k)
            if (w[k] != L.head[k]) reason = k + 1;                  // the first differing word wins
        const long long ns = (long long)(((unsigned long long)w[13] << 32) | w[12]);
        if (reason == 0 && ns < 0) reason = STATE_BAD_N_SAMPLES;
        odd = reason == 0 && (ns & 7) != 0;
    }
    const unsigned bad = __ballot_sync(0xffffffffu, reason != 0);
    const unsigned un = __ballot_sync(0xffffffffu, odd);
    const int lane = threadIdx.x & 31;
    if (bad) {
        const int fl = __ffs(bad) - 1;
        const int fr = __shfl_sync(0xffffffffu, reason, fl);
        if (lane == 0) {
            atomicAdd(&out->bad, (unsigned)__popc(bad));
            atomicMin(&out->first, ((unsigned long long)(r - lane + fl) << 8) | (unsigned long long)fr);
        }
    }
    if (un && lane == 0) atomicOr(&out->unaligned, 1u);
}

}  // namespace pb
