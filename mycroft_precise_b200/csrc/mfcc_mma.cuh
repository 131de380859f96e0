// mfcc_mma.cuh -- the stateful MFCC tick (n_fft 512 = frame, hop >= 512, chunk >= hop) with the DFT as fp16 matrix products on
// mma.sync m16n8k16, in the decomposition of mfcc_tc.cuh / mfcc_tc3.cuh (n = n2 + 32 q, k = 16 m + r):
//   stage 1  Y_r[n2] = sum_q d[n2 + 32 q] w16^(q r), d = x - x0 = 256 hi + lo exactly in fp16, weights as hi / lo pieces
//            (four passes; TC_STAGE1 = false: radix-16 butterflies on the CUDA cores instead)
//   stage 2  Z_r = 2^-5 Y_r w512^(n2 r) as fp16 hi / lo rows (block r, frame), times one 64 x 64 matrix (three passes)
//   epilogue power (X[0] += 512 x0), mel sums, log, DCT, c0, ring row.
// A warp owns 8 frames per tile; mfcc_mma_plan_kernel builds the tick's frame list.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "mfcc_kernels.cuh"   // StreamState, MelTables, frames_ready, K1_EPS
#include "mfcc_tc.cuh"        // rdft16_x2

namespace pb {

constexpr int MM_FRAMES = 8;                    // frames per warp tile
constexpr int MM_WARPS = 6;
constexpr int MM_THREADS = 32 * MM_WARPS;
constexpr int MM_ZROWS = 10 * MM_FRAMES;        // stage-2 rows (block r, frame); r = 9 is zero padding of the last M tile
constexpr int MM_ZS = 72;                       // halves per stage-2 row (64 + 8: conflict-free fragment loads)
constexpr int MM_PLAN_THREADS = 256;
constexpr int MM_MAX_FILT = 32;                 // one filter per lane in the epilogue

struct __align__(16) MmRec {           // one frame completed by this tick
    const int16_t* frame;              // sample 0 of the frame in chunk coordinates; nullptr: padding
    int16_t* tail;                     // the stream's tail (the frame's first 8 len0c samples; receives the new tail)
    float* row;                        // the frame's MFCC ring row
    unsigned int pad;
    unsigned char len0c;               // 16-byte chunks of the frame that come from the tail
    unsigned char tail_nv;             // first frame of a stream only: 16-byte chunks of the new tail (0: nothing to copy)
    unsigned short tail_delta;         // ... which starts 8 tail_delta samples after `frame`
};
static_assert(sizeof(MmRec) == 32, "frame records are 32 bytes");

struct MmTables {                      // device pointers
    const uint2* b1;                   // stage-1 B fragments [var 4][ntile 2][lane 32]: 256 w_hi, 256 w_lo, w_hi, w_lo
    const uint2* b2;                   // stage-2 B fragments [piece 2][kstep 4][ntile 8][lane 32]
    const float2* tw;                  // [n2 32][r 9]: 2^-5 (cos, -sin)(2 pi n2 r / 512)
    float pscale;                      // |X|^2 of the scaled accumulators -> power of audio / 32768, divided by n_fft
};

// ---------------------------------------------------------------------------------------------------------------------
// Host tables (fragment order of mma.m16n8k16: b0 = B[2t, 2t + 1][g], b1 = B[2t + 8, 2t + 9][g], g = lane / 4, t = lane % 4)
static inline uint32_t mm_pack(__half lo, __half hi) {
    uint16_t a, b;
    memcpy(&a, &lo, 2); memcpy(&b, &hi, 2);
    return (uint32_t)a | ((uint32_t)b << 16);
}
static inline void mm_build_tables(std::vector<uint2>& b1, std::vector<uint2>& b2, std::vector<float2>& tw) {
    const double PI2 = 6.283185307179586476925286766559;
    auto w1 = [&](int q, int c) -> double {            // stage 1: column c = Y_0, Y_8, Re Y_1, Im Y_1, ...
        if (c == 0) return 1.0;
        if (c == 1) return (q & 1) ? -1.0 : 1.0;
        const double a = PI2 * ((q * (c >> 1)) & 15) / 16.0;
        return (c & 1) ? -sin(a) : cos(a);
    };
    auto piece = [](double v, int var) {                // var 0 / 1: hi / lo of 256 w; 2 / 3: hi / lo of w
        const __half h = __float2half_rn((float)v);
        const __half l = __float2half_rn((float)(v - (double)__half2float(h)));
        const __half p = (var & 1) ? l : h;
        return var < 2 ? __float2half_rn(256.f * __half2float(p)) : p;          // exact: a power of two
    };
    b1.assign(4 * 2 * 32, make_uint2(0u, 0u));
    for (int var = 0; var < 4; ++var)
        for (int nt = 0; nt < 2; ++nt)
            for (int lane = 0; lane < 32; ++lane) {
                const int g = lane >> 2, t = lane & 3, c = 8 * nt + g;
                b1[(var * 2 + nt) * 32 + lane] = make_uint2(mm_pack(piece(w1(2 * t, c), var), piece(w1(2 * t + 1, c), var)),
                                                             mm_pack(piece(w1(2 * t + 8, c), var), piece(w1(2 * t + 9, c), var)));
            }
    auto w2 = [&](int k, int n) -> double {             // stage 2: K = 2 n2 + im, N = quarter 16 + m (mfcc_tc.cuh)
        const int n2 = k >> 1, im = k & 1, quarter = n >> 4, m = n & 15;
        const double a = PI2 * n2 * (quarter < 2 ? m : m + 1) / 32.0;
        const double tr = cos(a), ti = -sin(a);
        if (quarter == 0) return im ? -ti : tr;
        if (quarter == 1) return im ? tr : ti;
        if (quarter == 2) return im ? ti : tr;
        return im ? -tr : ti;
    };
    auto piece2 = [](double v, int p) {
        const __half h = __float2half_rn((float)v);
        return p ? __float2half_rn((float)(v - (double)__half2float(h))) : h;
    };
    b2.assign(2 * 4 * 8 * 32, make_uint2(0u, 0u));
    for (int p = 0; p < 2; ++p)
        for (int ks = 0; ks < 4; ++ks)
            for (int nt = 0; nt < 8; ++nt)
                for (int lane = 0; lane < 32; ++lane) {
                    const int g = lane >> 2, t = lane & 3, n = 8 * nt + g, k = 16 * ks + 2 * t;
                    b2[((p * 4 + ks) * 8 + nt) * 32 + lane] = make_uint2(mm_pack(piece2(w2(k, n), p), piece2(w2(k + 1, n), p)),
                                                                         mm_pack(piece2(w2(k + 8, n), p), piece2(w2(k + 9, n), p)));
                }
    tw.assign(32 * 9, make_float2(0.f, 0.f));
    for (int n2 = 0; n2 < 32; ++n2)
        for (int r = 0; r <= 8; ++r) {
            const double a = PI2 * n2 * r / 512.0;
            tw[n2 * 9 + r] = make_float2((float)(cos(a) / 32.0), (float)(-sin(a) / 32.0));
        }
}

// CPU model of one frame: the fragment tables read through the kernel's index arithmetic, same splits and bin assembly
// -> |X[k]|^2 of the raw samples (pb_debug_mma_dft_power).
static inline float mm_half(uint32_t v, int upper) {
    const uint16_t u = (uint16_t)(upper ? v >> 16 : v & 0xffffu);
    __half h;
    memcpy(&h, &u, 2);
    return __half2float(h);
}
static inline float mm_f16(float v) { return __half2float(__float2half_rn(v)); }
static inline void mm_host_power(const int16_t* x, double* power) {
    static std::vector<uint2> b1, b2;
    static std::vector<float2> tw;
    if (b1.empty()) mm_build_tables(b1, b2, tw);
    static float w1[4][16][16], w2[2][64][64];                      // [var][q][c], [piece][k][n]
    for (int lane = 0; lane < 32; ++lane) {
        const int g = lane >> 2, t = lane & 3;
        for (int var = 0; var < 4; ++var)
            for (int nt = 0; nt < 2; ++nt) {
                const uint2 f = b1[(var * 2 + nt) * 32 + lane];
                const int c = 8 * nt + g;
                w1[var][2 * t][c] = mm_half(f.x, 0); w1[var][2 * t + 1][c] = mm_half(f.x, 1);
                w1[var][2 * t + 8][c] = mm_half(f.y, 0); w1[var][2 * t + 9][c] = mm_half(f.y, 1);
            }
        for (int p = 0; p < 2; ++p)
            for (int ks = 0; ks < 4; ++ks)
                for (int nt = 0; nt < 8; ++nt) {
                    const uint2 f = b2[((p * 4 + ks) * 8 + nt) * 32 + lane];
                    const int k = 16 * ks + 2 * t, n = 8 * nt + g;
                    w2[p][k][n] = mm_half(f.x, 0); w2[p][k + 1][n] = mm_half(f.x, 1);
                    w2[p][k + 8][n] = mm_half(f.y, 0); w2[p][k + 9][n] = mm_half(f.y, 1);
                }
    }
    const int x0 = x[0];
    float z[2][9][64];
    for (int n2 = 0; n2 < 32; ++n2) {
        float y[16];
        for (int c = 0; c < 16; ++c) {
            float acc = 0.f;
            for (int pass = 0; pass < 4; ++pass)                         // lo w_lo, lo w_hi, hi 256 w_lo, hi 256 w_hi
                for (int q = 0; q < 16; ++q) {
                    const int dv = (int)x[n2 + 32 * q] - x0, lo = ((dv & 255) ^ 128) - 128, hi = (dv - lo) >> 8;
                    acc += (float)(pass < 2 ? lo : hi) * w1[3 - pass][q][c];
                }
            y[c] = acc;
        }
        for (int r = 0; r <= 8; ++r) {
            const float yr = r == 0 ? y[0] : r == 8 ? y[1] : y[2 * r], yi = (r == 0 || r == 8) ? 0.f : y[2 * r + 1];
            const float2 w = tw[n2 * 9 + r];
            const float zr = fmaf(yr, w.x, -(yi * w.y)), zi = fmaf(yr, w.y, yi * w.x);
            const float hr = mm_f16(zr), hi = mm_f16(zi);
            z[0][r][2 * n2] = hr; z[0][r][2 * n2 + 1] = hi;
            z[1][r][2 * n2] = mm_f16(zr - hr); z[1][r][2 * n2 + 1] = mm_f16(zi - hi);
        }
    }
    for (int r = 0; r <= 8; ++r) {
        float X[64];
        for (int n = 0; n < 64; ++n) {
            float acc = 0.f;
            for (int k = 0; k < 64; ++k) acc += z[1][r][k] * w2[0][k][n] + z[0][r][k] * w2[1][k][n] + z[0][r][k] * w2[0][k][n];
            X[n] = acc;
        }
        for (int m = 0; m < 16; ++m) {
            const double re = X[m], im = X[16 + m], re2 = X[32 + m], im2 = X[48 + m];
            if (r == 0) {
                if (m == 0) power[0] = (re + 16.0 * x0) * (re + 16.0 * x0) * 1024.0;
                else power[16 * m] = (re * re + im * im) * 1024.0;
                if (m == 15) power[256] = re2 * re2 * 1024.0;
            } else {
                power[16 * m + r] = (re * re + im * im) * 1024.0;
                if (r < 8) power[16 * m + 16 - r] = (re2 * re2 + im2 * im2) * 1024.0;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// The frame list of a tick (Listener.update_vectors, network_runner.py:137-144); counters[parity] receives the frame count.
__global__ void __launch_bounds__(MM_PLAN_THREADS)
mfcc_mma_plan_kernel(const int16_t* __restrict__ pcm, const int* __restrict__ ids, int n, int chunk, int hop, StreamState st,
                     MmRec* __restrict__ recs, unsigned int* __restrict__ counters, int parity) {
    __shared__ int warp_tot[MM_PLAN_THREADS / 32];
    __shared__ unsigned int base_sh;
    constexpr int used = 512;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int i = blockIdx.x * MM_PLAN_THREADS + tid;
    int cnt = 0, d = 0, slot0 = 0, sid = 0;
    if (i < n) {
        sid = ids ? ids[i] : i;
        const long long n0 = st.n_samples[sid];
        const long long c0 = frames_ready(n0, used, hop);
        cnt = (int)(frames_ready(n0 + chunk, used, hop) - c0);
        d = (int)(c0 * hop - n0);
        slot0 = (int)(c0 % st.ring_rows);
        st.n_samples[sid] = n0 + chunk;
    }
    int incl = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    if (tid == 0) {
        int t = 0;
        for (int w = 0; w < MM_PLAN_THREADS / 32; ++w) { const int v = warp_tot[w]; warp_tot[w] = t; t += v; }
        base_sh = t ? atomicAdd(&counters[parity], (unsigned int)t) : 0u;
    }
    __syncthreads();
    if (i >= n) return;
    const unsigned int off0 = base_sh + warp_tot[warp] + (incl - cnt);
    const int16_t* chunk_p = pcm + (long long)i * chunk;
    const int tail_off = min(d + cnt * hop, chunk);
    for (int j = 0; j < cnt; ++j) {
        MmRec r;
        const int dj = d + j * hop;
        int sl = slot0 + j;
        if (sl >= st.ring_rows) sl -= st.ring_rows;
        r.frame = chunk_p + dj;
        r.tail = st.tail + (long long)sid * st.tail_cap;
        r.row = st.ring + ((long long)sid * st.ring_rows + sl) * st.row_stride;
        r.pad = 0u;
        r.len0c = (unsigned char)(dj < 0 ? min(used, -dj) >> 3 : 0);
        r.tail_nv = (unsigned char)(j == 0 ? (chunk - tail_off) >> 3 : 0);
        r.tail_delta = (unsigned short)(j == 0 ? (tail_off - dj) >> 3 : 0);
        int4* dst = reinterpret_cast<int4*>(recs + off0 + j);
        dst[0] = reinterpret_cast<const int4*>(&r)[0];
        dst[1] = reinterpret_cast<const int4*>(&r)[1];
    }
}

// ---------------------------------------------------------------------------------------------------------------------
struct MmWarp {
    union {
        int16_t x[MM_FRAMES][512];                       // the tile's samples
        float p[MM_FRAMES][260];                         // ... then the power spectra
    } u;
    __half z[2][MM_ZROWS][MM_ZS];                        // stage-2 operand, pieces hi / lo
    float lg[MM_FRAMES][MM_MAX_FILT + 1];
    MmRec rec[MM_FRAMES];
};
struct MmSmem {
    uint2 b2[2 * 4 * 8 * 32];
    float2 tw[32 * 9];
    MmWarp w[MM_WARPS];
};

__device__ __forceinline__ void mm_mma(float (&d)[4], const uint32_t (&a)[4], uint2 b) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b.x), "r"(b.y));
}
__device__ __forceinline__ uint32_t mm_h2(float a, float b) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}
// Z = Y * tw (complex), stored as fp16 hi / lo pieces at (row, K = 2 n2, 2 n2 + 1)
__device__ __forceinline__ void mm_put_z(MmWarp& w, int row, int n2, float yr, float yi, float2 tw) {
    const float zr = fmaf(yr, tw.x, -(yi * tw.y)), zi = fmaf(yr, tw.y, yi * tw.x);
    const __half2 hi = __floats2half2_rn(zr, zi);
    const float2 hf = __half22float2(hi);
    const __half2 lo = __floats2half2_rn(zr - hf.x, zi - hf.y);
    *reinterpret_cast<__half2*>(&w.z[0][row][2 * n2]) = hi;
    *reinterpret_cast<__half2*>(&w.z[1][row][2 * n2]) = lo;
}

// TC_STAGE1: stage 1 on the tensor cores (k1 mode 5), else on the CUDA cores (k1 mode 4).  SHFL_EPI: the DCT reads the log-mels
// by shuffles instead of shared memory (k1 mode 6).
template <bool TC_STAGE1, bool SHFL_EPI>
__global__ void __launch_bounds__(MM_THREADS, 1)
mfcc_mma_kernel(MmTables tab, MelTables mt, const MmRec* __restrict__ recs, unsigned int* __restrict__ counters, int parity) {
    extern __shared__ __align__(16) unsigned char mm_raw[];
    MmSmem& sm = *reinterpret_cast<MmSmem*>(mm_raw);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    for (int e = tid; e < 2 * 4 * 8 * 32; e += MM_THREADS) sm.b2[e] = __ldg(tab.b2 + e);
    for (int e = tid; e < 32 * 9; e += MM_THREADS) sm.tw[e] = __ldg(tab.tw + e);
    MmWarp& w = sm.w[warp];
    for (int e = lane; e < 2 * MM_FRAMES * MM_ZS / 2; e += 32) {                // rows of the padding block r = 9 stay zero
        const int p = e / (MM_FRAMES * MM_ZS / 2), o = e % (MM_FRAMES * MM_ZS / 2);
        reinterpret_cast<uint32_t*>(&w.z[p][9 * MM_FRAMES][0])[o] = 0u;
    }
    uint2 b1[4][2];
    if (TC_STAGE1) {
#pragma unroll
        for (int v = 0; v < 4; ++v)
#pragma unroll
            for (int nt = 0; nt < 2; ++nt) b1[v][nt] = __ldg(tab.b1 + (v * 2 + nt) * 32 + lane);
    }
    const int n_frames = (int)*reinterpret_cast<volatile unsigned int*>(&counters[parity]);
    __syncthreads();
    if (blockIdx.x == 0 && tid == 0) counters[parity ^ 1] = 0u;      // the next tick's plan kernel counts from zero
    const int n_filt = mt.n_filt, n_out = mt.n_out;
    const int n_tiles = (n_frames + MM_FRAMES - 1) / MM_FRAMES;

    for (int tile = blockIdx.x * MM_WARPS + warp; tile < n_tiles; tile += gridDim.x * MM_WARPS) {
        // ---- records, samples (tail part first), new tails
        if (lane < MM_FRAMES) {
            const int idx = tile * MM_FRAMES + lane;
            int4 a = make_int4(0, 0, 0, 0), b = make_int4(0, 0, 0, 0);
            if (idx < n_frames) {
                const int4* p = reinterpret_cast<const int4*>(recs + idx);
                a = __ldg(p); b = __ldg(p + 1);
            }
            reinterpret_cast<int4*>(&w.rec[lane])[0] = a;
            reinterpret_cast<int4*>(&w.rec[lane])[1] = b;
        }
        __syncwarp();
        for (int e = lane; e < MM_FRAMES * 64; e += 32) {
            const int f = e >> 6, c = e & 63;
            const MmRec& r = w.rec[f];
            uint4 v = make_uint4(0u, 0u, 0u, 0u);
            if (r.frame != nullptr) v = *reinterpret_cast<const uint4*>((c < (int)r.len0c ? r.tail : r.frame) + 8 * c);
            *reinterpret_cast<uint4*>(&w.u.x[f][8 * c]) = v;
        }
        __syncwarp();                                    // every read of an old tail is done
        for (int f = 0; f < MM_FRAMES; ++f) {
            const MmRec& r = w.rec[f];
            if (r.frame == nullptr || r.tail_nv == 0) continue;
            const uint4* src = reinterpret_cast<const uint4*>(r.frame + 8 * (int)r.tail_delta);
            for (int c = lane; c < (int)r.tail_nv; c += 32) reinterpret_cast<uint4*>(r.tail)[c] = src[c];
        }

        // ---- stage 1 + twiddle -> stage-2 operand
        if (TC_STAGE1) {
#pragma unroll 1
            for (int f = 0; f < MM_FRAMES; ++f) {
                const int x0 = w.u.x[f][0];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    uint32_t ah[4], al[4];
#pragma unroll
                    for (int e = 0; e < 4; ++e) {                // fragment register e: row g (+8 for e odd), K 2t (+8 for e >= 2)
                        const int n2 = 16 * h + g + 8 * (e & 1), q = 2 * t + 8 * (e >> 1);
                        int hv[2], lv[2];
#pragma unroll
                        for (int j = 0; j < 2; ++j) {
                            const int dv = (int)w.u.x[f][n2 + 32 * (q + j)] - x0;
                            lv[j] = ((dv & 255) ^ 128) - 128;
                            hv[j] = (dv - lv[j]) >> 8;
                        }
                        ah[e] = mm_h2((float)hv[0], (float)hv[1]);
                        al[e] = mm_h2((float)lv[0], (float)lv[1]);
                    }
                    float acc[2][4];
#pragma unroll
                    for (int nt = 0; nt < 2; ++nt) {
                        acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
                        mm_mma(acc[nt], al, b1[3][nt]);
                        mm_mma(acc[nt], al, b1[2][nt]);
                        mm_mma(acc[nt], ah, b1[1][nt]);
                        mm_mma(acc[nt], ah, b1[0][nt]);
                    }
#pragma unroll
                    for (int half = 0; half < 2; ++half) {
                        const int n2 = 16 * h + g + 8 * half;
                        const float2* twr = &sm.tw[n2 * 9];
#pragma unroll
                        for (int nt = 0; nt < 2; ++nt) {
                            const float y0 = acc[nt][2 * half], y1 = acc[nt][2 * half + 1];
                            if (nt == 0 && t == 0) {             // columns 0, 1: Y_0, Y_8 (real)
                                mm_put_z(w, f, n2, y0, 0.f, twr[0]);
                                mm_put_z(w, 8 * MM_FRAMES + f, n2, y1, 0.f, twr[8]);
                            } else {
                                const int r = 4 * nt + t;
                                mm_put_z(w, r * MM_FRAMES + f, n2, y0, y1, twr[r]);
                            }
                        }
                    }
                }
            }
        } else {
#pragma unroll 1
            for (int it = lane; it < MM_FRAMES * 32; it += 32) {
                const int f = it >> 5, n2 = it & 31;
                const int x0 = w.u.x[f][0];
                float in[16], yr[9], yi[9];
#pragma unroll
                for (int q = 0; q < 16; ++q) in[q] = (float)((int)w.u.x[f][n2 + 32 * q] - x0);
                rdft16_x2(in, yr, yi);                           // 2 Y
#pragma unroll
                for (int r = 0; r <= 8; ++r) mm_put_z(w, r * MM_FRAMES + f, n2, 0.5f * yr[r], 0.5f * yi[r], sm.tw[n2 * 9 + r]);
            }
        }
        const float x0g = (float)w.u.x[g][0];                   // first sample of frame g (the frame of this lane's stage-2 rows)
        __syncwarp();                                            // stage-2 operand complete; samples no longer needed

        // ---- stage 2 + power: M tile mt2 = blocks 2 mt2 (rows g) and 2 mt2 + 1 (rows g + 8), frame g
#pragma unroll 1
        for (int mt2 = 0; mt2 < 5; ++mt2) {
            float acc[8][4];
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
                uint32_t ah[4], al[4];
                const int ra = 16 * mt2 + g, k0 = 16 * ks + 2 * t;
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int row = ra + 8 * (e & 1), k = k0 + 8 * (e >> 1);
                    ah[e] = *reinterpret_cast<const uint32_t*>(&w.z[0][row][k]);
                    al[e] = *reinterpret_cast<const uint32_t*>(&w.z[1][row][k]);
                }
#pragma unroll
                for (int nt = 0; nt < 8; ++nt) {
                    const uint2 bh = sm.b2[((0 * 4 + ks) * 8 + nt) * 32 + lane], bl = sm.b2[((1 * 4 + ks) * 8 + nt) * 32 + lane];
                    mm_mma(acc[nt], al, bh);
                    mm_mma(acc[nt], ah, bl);
                    mm_mma(acc[nt], ah, bh);
                }
            }
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                const int r = 2 * mt2 + half;
                if (r > 8) continue;
#pragma unroll
                for (int ntp = 0; ntp < 2; ++ntp)
#pragma unroll
                    for (int j = 0; j < 2; ++j) {
                        const int m = 8 * ntp + 2 * t + j, e = 2 * half + j;
                        float re = acc[ntp][e];
                        const float im = acc[ntp + 2][e];
                        if (r == 0) {                            // X[16 m]: real only for m = 0
                            if (m == 0) w.u.p[g][0] = fmaf(16.f, x0g, re) * fmaf(16.f, x0g, re);   // X[0] += 2^-5 * 512 x0
                            else w.u.p[g][16 * m] = fmaf(im, im, re * re);
                        } else {
                            w.u.p[g][16 * m + r] = fmaf(im, im, re * re);
                        }
                        const float re2 = acc[ntp + 4][e], im2 = acc[ntp + 6][e];
                        if (r == 0) {
                            if (m == 15) w.u.p[g][256] = re2 * re2;
                        } else if (r < 8) {
                            w.u.p[g][16 * m + 16 - r] = fmaf(im2, im2, re2 * re2);
                        }
                    }
            }
        }
        __syncwarp();

        // ---- epilogue: mel sums, log, DCT, c0, ring rows
#pragma unroll 1
        for (int f = 0; f < MM_FRAMES; ++f) {
            const MmRec& r = w.rec[f];
            if (r.frame == nullptr) continue;                    // padding frames are at the end: uniform over the warp
            float tot = 0.f;
            for (int k = lane; k < 257; k += 32) tot += w.u.p[f][k];
#pragma unroll
            for (int o = 16; o >= 1; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
            float lgv = 0.f;
            if (lane < n_filt) {
                const int lo = __ldg(mt.grid + lane), mid = __ldg(mt.grid + lane + 1), hi = __ldg(mt.grid + lane + 2);
                float m0 = 0.f, m1 = 0.f;
                for (int k = lo; k < mid; ++k) m0 = fmaf(__ldg(mt.w_rise + k), w.u.p[f][k], m0);
                for (int k = mid; k < hi; ++k) m1 = fmaf(__ldg(mt.w_fall + k), w.u.p[f][k], m1);
                lgv = logf(fmaxf((m0 + m1) * tab.pscale, K1_EPS));
                if (!SHFL_EPI) w.lg[f][lane] = lgv;
            }
            __syncwarp();
            float v = 0.f;
            for (int j = 0; j < n_filt; ++j) {
                const float l = SHFL_EPI ? __shfl_sync(0xffffffffu, lgv, j) : w.lg[f][j];
                if (lane < n_out) v = fmaf(__ldg(mt.dct + lane * n_filt + j), l, v);
            }
            if (lane < n_out) r.row[lane] = lane == 0 ? logf(fmaxf(tot * tab.pscale, K1_EPS)) : v;
        }
        __syncwarp();                                            // the next tile overwrites samples, records and log-mels
    }
}

}  // namespace pb
