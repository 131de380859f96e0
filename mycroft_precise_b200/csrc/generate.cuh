// generate.cuh -- wake-word and not-wake-word clips overlaid on background recordings (pb_generate): the audio side of
// precise-train-generated's vectors_from_fn (precise/scripts/train_generated.py:118-190) on the device.
//
// Item i is the first len_i samples of a background at gain f, overlaid with a table of segments laid back to back from the
// item's sample 0: a segment is a stretch of one clip, or silence.  Where the host draws the pieces and cuts them into
// chunks, the kernel is a plain overlay.  With S the exact int64 sum of squares of a WHOLE recording (background or clip)
// over its raw int16 samples and n its length,
//     rms = S > 0 ? sqrt(S / n) : 0,   vol = f rms_bg,   g = rms_clip > 0 ? vol / rms_clip : 0 (0 in silence),
//     y = 0.4 (f x_bg) + 0.6 (g x_clip),   out = int16(clamp(rint(y), -32768, 32767))
// in IEEE double with every conversion, product, quotient, square root and sum rounded on its own (no FMA contraction), so
// the output is one function of the inputs that a numpy restatement reproduces bit for bit.
//
//   gen_sums_kernel    one CTA per (recording, GEN_SEG samples): per-thread int64 sums of x^2, a block reduction and one
//                      integer atomicAdd into the recording's sum, so the sums do not depend on the order the CTAs land.
//   gen_mix_kernel     one CTA per GEN_TILE samples of an item: the CTA finds its item and its first segment once, then walks
//                      the segments that overlap its tile, each thread a strided run of samples.  The stream goes to `out`
//                      (when given) and to `ws`, the aligned workspace K1 reads (when given).
//   gen_gather_kernel  one thread per (chosen window, row, feature): the window's n_features frame rows, as
//                      vectorize_gather_kernel copies a clip's, from the listener schedule's window table.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pb {

constexpr int GEN_THREADS = 256;
constexpr long long GEN_SEG = 1 << 16;       // samples per CTA of the sums
constexpr long long GEN_TILE = 1 << 13;      // samples per CTA of the mix
constexpr long long GEN_MAX_SEG = 1ll << 62;  // longest segment: positions within an item stay below 2^63

struct GenRec {                              // a recording whose sum of squares the mix needs
    long long src;                           // first sample (in the backgrounds or in the clips)
    long long len;
    int clip;                                // 0: a background, 1: a clip
    int pad;
};

struct GenItem {
    long long bg;                            // first sample of the background
    long long len;                           // samples generated
    long long out;                           // first sample in `out`
    long long ws;                            // first sample in `ws` (a multiple of 8)
    long long seg0, seg1;                    // its segments
    double f;                                // background gain
    int bg_rec;                              // the background's GenRec
    int pad;
};

struct GenSeg {
    long long pos;                           // first sample of the item it covers
    long long len;
    long long src;                           // first sample in the clips (silence: unused)
    int rec;                                 // the clip's GenRec, -1 for silence
    int pad;
};

// Largest j in [lo, hi) with a[j].pos <= v (a[lo].pos <= v).
__device__ __forceinline__ long long gen_find_seg(const GenSeg* __restrict__ s, long long lo, long long hi, long long v) {
    --hi;
    while (lo < hi) {
        const long long mid = (lo + hi + 1) >> 1;
        if (s[mid].pos <= v) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__device__ __forceinline__ int gen_find(const long long* __restrict__ a, int n, long long v) {
    int lo = 0, hi = n - 1;                  // last j with a[j] <= v
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(a + mid) <= v) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__device__ __forceinline__ double gen_rms(unsigned long long s, long long n) {
    return s > 0 ? __dsqrt_rn(__ddiv_rn(__ull2double_rn(s), __ll2double_rn(n))) : 0.0;
}

__global__ void __launch_bounds__(GEN_THREADS) gen_sums_kernel(const int16_t* __restrict__ bg, const int16_t* __restrict__ clips,
                                                               const GenRec* __restrict__ recs, const long long* __restrict__ seg0,
                                                               int n_recs, unsigned long long* __restrict__ sums) {
    const long long b = blockIdx.x;
    const int r = gen_find(seg0, n_recs, b);
    const GenRec rc = recs[r];
    const int16_t* x = (rc.clip ? clips : bg) + rc.src;
    const long long k0 = (b - seg0[r]) * GEN_SEG, k1 = min(rc.len, k0 + GEN_SEG);
    long long s = 0;
    for (long long k = k0 + threadIdx.x; k < k1; k += GEN_THREADS) {
        const long long v = x[k];
        s += v * v;
    }
    __shared__ long long red[GEN_THREADS / 32];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        long long t = 0;
        for (int j = 0; j < GEN_THREADS / 32; ++j) t += red[j];
        atomicAdd(&sums[r], (unsigned long long)t);
    }
}

__global__ void __launch_bounds__(GEN_THREADS) gen_mix_kernel(const int16_t* __restrict__ bg, const int16_t* __restrict__ clips,
                                                              const GenRec* __restrict__ recs, const unsigned long long* __restrict__ sums,
                                                              const GenItem* __restrict__ items, const long long* __restrict__ tile0,
                                                              int n_items, const GenSeg* __restrict__ segs,
                                                              int16_t* __restrict__ out, int16_t* __restrict__ ws) {
    const long long b = blockIdx.x;
    const int i = gen_find(tile0, n_items, b);
    const GenItem it = items[i];
    const long long k0 = (b - tile0[i]) * GEN_TILE, k1 = min(it.len, k0 + GEN_TILE);
    const double vol = __dmul_rn(it.f, gen_rms(sums[it.bg_rec], recs[it.bg_rec].len));
    for (long long j = gen_find_seg(segs, it.seg0, it.seg1, k0); j < it.seg1; ++j) {
        const GenSeg sg = segs[j];
        if (sg.pos >= k1) break;
        const long long a = max(k0, sg.pos), e = min(k1, sg.pos + sg.len);
        double g = 0.0;
        if (sg.rec >= 0) {
            const double r = gen_rms(sums[sg.rec], recs[sg.rec].len);
            g = r > 0.0 ? __ddiv_rn(vol, r) : 0.0;
        }
        const int16_t* xc = sg.rec >= 0 ? clips + sg.src - sg.pos : nullptr;
        for (long long k = a + threadIdx.x; k < e; k += GEN_THREADS) {
            const double xb = bg[it.bg + k], xs = xc ? (double)xc[k] : 0.0;
            const double y = rint(__dadd_rn(__dmul_rn(0.4, __dmul_rn(it.f, xb)), __dmul_rn(0.6, __dmul_rn(g, xs))));
            const int16_t v = (int16_t)(int)fmin(fmax(y, -32768.0), 32767.0);
            if (out) out[it.out + k] = v;
            if (ws) ws[it.ws + k] = v;
        }
    }
}

// wins [n]: the chosen windows' indices in the window table `starts`.
__global__ void gen_gather_kernel(const float* __restrict__ frames, const long long* __restrict__ starts,
                                  const long long* __restrict__ wins, int row_stride, int T, int F, long long n,
                                  float* __restrict__ out) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n * T * F) return;
    const int f = (int)(e % F);
    const long long q = e / F;
    const int t = (int)(q % T);
    const long long r = q / T;
    out[e] = frames[(starts[wins[r]] + t) * row_stride + f];
}

}  // namespace pb
