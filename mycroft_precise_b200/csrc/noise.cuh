// noise.cuh -- background noise mixed into clips (pb_add_noise): precise-add-noise's NoiseData.noised_audio
// (precise/scripts/add_noise.py:56-90) on the device.
//
// Item i is a clip with a ratio r.  Its noise span is the corpus read cyclically from the item's start position, one noise
// sample per clip sample.  The mix is
//     g = Sn > 0 ? r sqrt(Sa) / sqrt(Sn) : 0,   y = (1 - r) x + g n,   out = int16(clamp(trunc(y), -32768, 32767))
// with Sa = sum x^2 over the clip and Sn = sum n^2 over its span, both over the raw int16 samples (the reference's 1 / 32767
// scale cancels in the ratio and in its save_audio).  The sums are int64, so they are exact and do not depend on the order
// in which the segments' atomics land; y is IEEE double with every product and sum rounded on its own (no FMA contraction),
// so the output is one function of (clip, span, r) that a numpy restatement reproduces bit for bit.
//
//   noise_sums_kernel  one CTA per (item, segment of NZ_SEG samples): per-thread int64 sums of x^2 and n^2, a block reduction,
//                      and one integer atomicAdd per sum into the item's pair.  A long recording spreads over many CTAs.
//   noise_mix_kernel   the same grid: the item's gain from its sums, then y per sample.  The whole clip goes to `out` (when
//                      given) and its last `crop` samples to `crop_out`, the aligned workspace pb_vectorize_clips' K1 reads.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pb {

constexpr int NZ_THREADS = 256;
constexpr long long NZ_SEG = 1 << 16;        // samples per CTA

struct NoiseItem {
    long long src;       // first sample of the clip in the recordings
    long long len;       // samples
    long long npos;      // noise position of the clip's sample 0, in [0, n_noise)
    long long out;       // first sample of the clip in `out`
    long long crop_out;  // first sample of the clip's last `crop` samples in `crop_out`
    long long crop;      // samples of the clip that go to `crop_out` (its last ones)
    double r;            // noise ratio in [0, 1]
};

// The item and segment of CTA b: seg0 [n_items + 1] is the exclusive prefix of each item's segment count.
__device__ __forceinline__ int nz_find_item(const long long* __restrict__ seg0, int n_items, long long b) {
    int lo = 0, hi = n_items - 1;
    while (lo < hi) {                        // last item whose seg0 <= b
        const int mid = (lo + hi + 1) >> 1;
        if (seg0[mid] <= b) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__device__ __forceinline__ long long nz_wrap(long long p, long long n_noise) { return p < n_noise ? p : p % n_noise; }

// The noise index of a thread's samples k, k + NZ_THREADS, ...: one division at the start, then a step and one subtraction.
struct NzCursor {
    long long idx, step, n;
    __device__ __forceinline__ NzCursor(long long npos, long long k, long long n_noise)
        : idx(nz_wrap(npos + k, n_noise)), step(nz_wrap(NZ_THREADS, n_noise)), n(n_noise) {}
    __device__ __forceinline__ void next() { idx += step; if (idx >= n) idx -= n; }
};

__global__ void __launch_bounds__(NZ_THREADS) noise_sums_kernel(const int16_t* __restrict__ pcm, const int16_t* __restrict__ noise,
                                                                long long n_noise, const NoiseItem* __restrict__ items,
                                                                const long long* __restrict__ seg0, int n_items,
                                                                unsigned long long* __restrict__ sums) {
    const long long b = blockIdx.x;
    const int i = nz_find_item(seg0, n_items, b);
    const NoiseItem it = items[i];
    const long long k0 = (b - seg0[i]) * NZ_SEG, k1 = min(it.len, k0 + NZ_SEG);
    long long sa = 0, sn = 0;
    NzCursor c(it.npos, k0 + threadIdx.x, n_noise);
    for (long long k = k0 + threadIdx.x; k < k1; k += NZ_THREADS, c.next()) {
        const long long x = pcm[it.src + k], n = noise[c.idx];
        sa += x * x;
        sn += n * n;
    }
    __shared__ long long red[2][NZ_THREADS / 32];
    for (int o = 16; o > 0; o >>= 1) {
        sa += __shfl_xor_sync(0xffffffffu, sa, o);
        sn += __shfl_xor_sync(0xffffffffu, sn, o);
    }
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { red[0][w] = sa; red[1][w] = sn; }
    __syncthreads();
    if (threadIdx.x == 0) {
        long long ta = 0, tn = 0;
        for (int j = 0; j < NZ_THREADS / 32; ++j) { ta += red[0][j]; tn += red[1][j]; }
        atomicAdd(&sums[2 * i], (unsigned long long)ta);
        atomicAdd(&sums[2 * i + 1], (unsigned long long)tn);
    }
}

__global__ void __launch_bounds__(NZ_THREADS) noise_mix_kernel(const int16_t* __restrict__ pcm, const int16_t* __restrict__ noise,
                                                               long long n_noise, const NoiseItem* __restrict__ items,
                                                               const long long* __restrict__ seg0, int n_items,
                                                               const unsigned long long* __restrict__ sums,
                                                               int16_t* __restrict__ out, int16_t* __restrict__ crop_out) {
    const long long b = blockIdx.x;
    const int i = nz_find_item(seg0, n_items, b);
    const NoiseItem it = items[i];
    const long long k0 = (b - seg0[i]) * NZ_SEG, k1 = min(it.len, k0 + NZ_SEG);
    const long long c0 = it.len - it.crop;                  // first sample that goes to crop_out
    const long long kb = out ? k0 : max(k0, c0);            // without out, only the cropped tail is mixed
    if (kb >= k1) return;
    const unsigned long long sa = sums[2 * i], sn = sums[2 * i + 1];
    const double g = sn > 0 ? __ddiv_rn(__dmul_rn(it.r, __dsqrt_rn((double)sa)), __dsqrt_rn((double)sn)) : 0.0;
    const double q = 1.0 - it.r;
    NzCursor c(it.npos, kb + threadIdx.x, n_noise);
    for (long long k = kb + threadIdx.x; k < k1; k += NZ_THREADS, c.next()) {
        const double x = pcm[it.src + k], n = noise[c.idx];
        const double y = trunc(__dadd_rn(__dmul_rn(q, x), __dmul_rn(g, n)));
        const int16_t v = (int16_t)(int)fmin(fmax(y, -32768.0), 32767.0);
        if (out) out[it.out + k] = v;
        if (crop_out && k >= c0) crop_out[it.crop_out + (k - c0)] = v;
    }
}

}  // namespace pb
