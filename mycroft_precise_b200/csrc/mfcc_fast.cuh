// mfcc_fast.cuh -- K1 fast path: warp-autonomous MFCC pipeline for the 16-byte-aligned geometry
// (n_fft = window-crop = 512 samples; hop, chunk and buffer length multiples of 8 samples -- true for
// the reference defaults, precise/params.py:140-144, and the 1024-sample runner chunk).
//
// Every warp is its own pipeline, there is no block-level barrier after start-up:
//
//   pass p:  [bulk copy of pass p+1's two frames -> staging buffer (p+1)&1, cp.async.bulk + mbarrier]
//            wait for buffer p&1 -> 16 x LDS.32 per lane -> FFT-512 (fft512.cuh; the same buffer is
//            reused as the transpose scratch and then holds the 257 power bins) -> mel/log/DCT by the
//            16 lanes of the half-warp -> one coalesced store of the MFCC row
//
// Mel stage on 16 lanes.  The spectrum is cut into "pieces" (<= 8 bins, never crossing a mel-grid
// point; built on the host).  Lane l accumulates pieces l, l+16, ...: rise/fall partial sums
// (w_rise[k] P[k], w_fall[k] P[k]) and its share of the total power.  Filter j then adds the rise
// partials of grid segment j and the fall partials of segment j+1 (sonopy.filterbanks geometry, see
// mfcc_kernels.cuh), takes log(max(., eps)), and lane c forms DCT row c.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "fft512.cuh"
#include "mfcc_kernels.cuh"

namespace pb {

// ------------------------------------------------------------------------------------------------
// PTX: mbarrier + 1-D bulk async copy (TMA engine, SASS UBLKCP)
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    } while (!ok);
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// ------------------------------------------------------------------------------------------------
constexpr int K1F_THREADS = 128;
constexpr int K1F_WARPS = K1F_THREADS / 32;
constexpr int K1F_MAX_PIECES = 128;
constexpr int K1F_PIECE_LEN = 8;
constexpr int K1F_STREAMS_PER_WARP = 16;
constexpr int K1F_MAX_NEW = 8;
constexpr int K1F_BUF_ELEMS = XCH_ELEMS + 8;   // +64 B: the two half-warps of a warp hit disjoint bank halves on 32-bit accesses

constexpr int K1F_PART = 132;                  // per frame: rise partials [0,64), fall partials [64,128), [128] = 0
constexpr int K1F_ZERO_BIN = 260;              // a bin slot that always reads 0 (padding entries of the piece table)

struct FastTables {            // device copies built by the host (api.cu)
    const float4* ptab;        // [npl][8][16]  (byte offset of the bin in P, w_rise, w_fall, -) for piece p = lane + 16 q, entry e
    const unsigned char* ctab; // [n_filt][maxc] indices into the partial array (128 = zero slot)
    const float* dct_t;        // [n_filt][16 * nol]  DCT rows transposed: dct_t[j][c]
    int npl, maxc, nol;
};

struct K1FWarp {               // per warp
    float2 buf[2][2][K1F_BUF_ELEMS];           // [stage][half]: input staging -> transpose scratch -> power bins
    float part[2][K1F_PART];
    float mel[2][K1_MAX_FILT];
    unsigned long long bar[2];
    // stream mode bookkeeping for the warp's tile of streams
    long long st_n0[K1F_STREAMS_PER_WARP], st_ts0[K1F_STREAMS_PER_WARP], st_c0[K1F_STREAMS_PER_WARP];
    int st_id[K1F_STREAMS_PER_WARP], st_cnt[K1F_STREAMS_PER_WARP];
    short fr_stream[K1F_STREAMS_PER_WARP * K1F_MAX_NEW], fr_sub[K1F_STREAMS_PER_WARP * K1F_MAX_NEW];
};

// shared-memory copies of the tables: [ptab | dct_t | ctab], carved from the dynamic tail
struct K1FTab {
    const float4* ptab;
    const float* dct_t;
    const unsigned char* ctab;
};

__device__ __forceinline__ K1FTab load_fast_tables(unsigned char* smem, const MelTables& t, const FastTables& ft) {
    float4* sp = reinterpret_cast<float4*>(smem);
    const int np = ft.npl * 128;
    float* sd = reinterpret_cast<float*>(sp + np);
    const int nd = t.mels_only ? 0 : t.n_filt * 16 * ft.nol;
    unsigned char* sc = reinterpret_cast<unsigned char*>(sd + nd);
    for (int k = threadIdx.x; k < np; k += blockDim.x) sp[k] = __ldg(ft.ptab + k);
    for (int k = threadIdx.x; k < nd; k += blockDim.x) sd[k] = __ldg(ft.dct_t + k);
    for (int k = threadIdx.x; k < t.n_filt * ft.maxc; k += blockDim.x) sc[k] = ft.ctab[k];
    K1FTab r;
    r.ptab = sp; r.dct_t = sd; r.ctab = sc;
    return r;
}

// mel / log / DCT for one frame by its 16 lanes, table driven and branch free.
//   P     : 257 power bins in shared memory; P[K1F_ZERO_BIN] must read 0
//   part  : K1F_PART floats of scratch; part[128] must read 0
//   eoff  : this lane's 8 entry offsets (in float4 units) into a piece-table block: ((i + rot) & 7) * 16 + l16
// All 32 lanes of the warp call this (the other half works on its own frame); `active` gates the store.
// UQ / UC unroll the piece and filter-slot loops: above 1, the shared loads of several iterations are in flight at once
// (piece entries, then the bins they select; slot indices, then the partials they select); every sum keeps its order.
template <int UQ = 1, int UC = 1>
__device__ __forceinline__ void mel16(const float* P, const K1FTab& tb, const FastTables& ft, const MelTables& t,
                                      float* part, float* mel, const int (&eoff)[8], int l16, bool active,
                                      float* __restrict__ out) {
    const char* Pb = reinterpret_cast<const char*>(P);
    float tot = 0.f;
#pragma unroll UQ
    for (int q = 0; q < ft.npl; ++q) {
        const float4* blk = tb.ptab + q * 128;
        float r = 0.f, f = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float4 e = blk[eoff[i]];
            const float pw = *reinterpret_cast<const float*>(Pb + __float_as_int(e.x));
            tot += pw;
            r = fmaf(e.y, pw, r);
            f = fmaf(e.z, pw, f);
        }
        part[q * 16 + l16] = r;
        part[64 + q * 16 + l16] = f;
    }
#pragma unroll
    for (int d = 8; d >= 1; d >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, d);
    __syncwarp();
#pragma unroll 1
    for (int j = l16; j < t.n_filt; j += 16) {
        const unsigned char* ci = tb.ctab + j * ft.maxc;
        float m0 = 0.f, m1 = 0.f;
#pragma unroll UC
        for (int c = 0; c + 1 < ft.maxc; c += 2) { m0 += part[ci[c]]; m1 += part[ci[c + 1]]; }
        if (ft.maxc & 1) m0 += part[ci[ft.maxc - 1]];
        mel[j] = logf(fmaxf(m0 + m1, K1_EPS));
    }
    __syncwarp();
    if (t.mels_only) {
        for (int j = l16; j < t.n_out; j += 16)
            if (active) out[j] = mel[j];
    } else {
        const int ld = 16 * ft.nol;
#pragma unroll 1
        for (int c = l16; c < t.n_out; c += 16) {
            float a0 = 0.f, a1 = 0.f;
            const float* d = tb.dct_t + c;
#pragma unroll 4
            for (int j = 0; j + 1 < t.n_filt; j += 2) { a0 = fmaf(d[j * ld], mel[j], a0); a1 = fmaf(d[(j + 1) * ld], mel[j + 1], a1); }
            if (t.n_filt & 1) a0 = fmaf(d[(t.n_filt - 1) * ld], mel[t.n_filt - 1], a0);
            const float v = c == 0 ? logf(fmaxf(tot, K1_EPS)) : a0 + a1;
            if (active) out[c] = v;
        }
    }
    __syncwarp();
}

// One FFT + mel pass for the warp's two frames whose 1 KB inputs have landed in ws.buf[stage].
__device__ __forceinline__ void fast_pass(K1FWarp& ws, int stage, uint32_t parity, const FftLaneConst& lc, const K1FTab& tb,
                                          const FastTables& ft, const MelTables& t, float scale, const int (&eoff)[8],
                                          int l16, int half, bool active, float* __restrict__ out) {
    mbar_wait(&ws.bar[stage], parity);
    const int* in = reinterpret_cast<const int*>(ws.buf[stage][half]);
    cpx z[16];
#pragma unroll
    for (int n1 = 0; n1 < 16; ++n1) {
        // int16 pair -> two floats without I2F (quarter-rate pipe): flip the sign bits (u = v + 32768), drop each half
        // into the mantissa of 2^23 and subtract 2^23 + 32768; exact.
        const unsigned v = (active ? (unsigned)in[16 * n1 + l16] : 0u) ^ 0x80008000u;
        z[n1].x = __uint_as_float(__byte_perm(v, 0x4b000000u, 0x7610)) - 8421376.f;
        z[n1].y = __uint_as_float(__byte_perm(v, 0x4b000000u, 0x7632)) - 8421376.f;
    }
    __syncwarp();                                  // all lanes have read the staged samples: the buffer becomes scratch
    float* P = reinterpret_cast<float*>(ws.buf[stage][half]);
    fft512_power(z, lc, ws.buf[stage][half], P, scale, l16, active);   // P aliases the scratch: written after the last scratch read
    if (l16 == 0) P[K1F_ZERO_BIN] = 0.f;           // padding entries of the piece table point here
    __syncwarp();
    mel16(P, tb, ft, t, ws.part[half], ws.mel[half], eoff, l16, active, out);
}

// ------------------------------------------------------------------------------------------------
// Stateless batch kernel (pb_mfcc on the aligned geometry).  Global frame g = stream * n_frames + f.
__global__ void __launch_bounds__(K1F_THREADS, 4)
mfcc_fast_batch_kernel(const int16_t* __restrict__ pcm, long long samples_per_stream, long long n_frames_per_stream,
                       long long total_frames, int hop, float scale, MelTables tab, FastTables ft, float* __restrict__ out) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    K1FWarp* wsm = reinterpret_cast<K1FWarp*>(smem_raw);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, l16 = lane & 15, half = lane >> 4;
    K1FWarp& ws = wsm[warp];
    const K1FTab tb = load_fast_tables(smem_raw + K1F_WARPS * sizeof(K1FWarp), tab, ft);
    if (lane == 0) { mbar_init(&ws.bar[0], 1); mbar_init(&ws.bar[1], 1); fence_mbar_init(); }
    if (l16 == 0) ws.part[half][128] = 0.f;
    int eoff[8];                                   // rotated walk through a piece: see mel16
    {
        const int rot = ((l16 >> 2) + (half << 2)) & 7;
#pragma unroll
        for (int i = 0; i < 8; ++i) eoff[i] = ((i + rot) & 7) * 16 + l16;
    }
    FftLaneConst lc;
    load_lane_const(lc, tab.tw_stage, tab.tw_post, l16);
    __syncthreads();

    const long long n_pairs = (total_frames + 1) / 2;
    const long long gwarp = (long long)blockIdx.x * K1F_WARPS + warp, nwarps = (long long)gridDim.x * K1F_WARPS;
    auto issue = [&](long long pair, int stage) {            // lane 0: bulk copies for both frames of `pair`
        const long long g0 = 2 * pair;
        const int nfr = (g0 + 1 < total_frames) ? 2 : 1;
        fence_proxy_async();
        mbar_expect_tx(&ws.bar[stage], 1024u * nfr);
        for (int hf = 0; hf < nfr; ++hf) {
            const long long g = g0 + hf, s = g / n_frames_per_stream, f = g - s * n_frames_per_stream;
            bulk_g2s(ws.buf[stage][hf], pcm + s * samples_per_stream + f * hop, 1024u, &ws.bar[stage]);
        }
    };
    long long pair = gwarp;
    int it = 0;
    if (pair < n_pairs && lane == 0) issue(pair, 0);
    for (; pair < n_pairs; pair += nwarps, ++it) {
        const int stage = it & 1;
        const long long next = pair + nwarps;
        if (next < n_pairs && lane == 0) issue(next, stage ^ 1);
        const long long g = 2 * pair + half;
        const bool active = g < total_frames;
        fast_pass(ws, stage, (uint32_t)((it >> 1) & 1), lc, tb, ft, tab, scale, eoff, l16, half, active,
                  out + (active ? g : 0) * tab.n_out);
    }
}

// ------------------------------------------------------------------------------------------------
// Stateful tick (pb_update / pb_update_vectors on the aligned geometry): a warp owns 16 streams.
// LEAN (opt-in, pb_debug_k1_mode 2; not yet validated on hardware): the per-pass set-up in 32-bit arithmetic.  The profile
// shows 16 % of this kernel's executed instructions in that set-up (a 64-bit modulo for the ring slot and 64-bit products
// for the source offsets, per frame); LEAN derives both from two per-stream ints computed once per tile
// (slot of the stream's first new frame, offset of that frame's first sample relative to the chunk).
template <bool LEAN>
__global__ void __launch_bounds__(K1F_THREADS, 4)
mfcc_fast_stream_kernel(const int16_t* __restrict__ pcm, const int* __restrict__ ids, int n, int chunk, int hop, int spw,
                        float scale, MelTables tab, FastTables ft, StreamState st) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    K1FWarp* wsm = reinterpret_cast<K1FWarp*>(smem_raw);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, l16 = lane & 15, half = lane >> 4;
    K1FWarp& ws = wsm[warp];
    const K1FTab tb = load_fast_tables(smem_raw + K1F_WARPS * sizeof(K1FWarp), tab, ft);
    if (lane == 0) { mbar_init(&ws.bar[0], 1); mbar_init(&ws.bar[1], 1); fence_mbar_init(); }
    if (l16 == 0) ws.part[half][128] = 0.f;
    int eoff[8];                                   // rotated walk through a piece: see mel16
    {
        const int rot = ((l16 >> 2) + (half << 2)) & 7;
#pragma unroll
        for (int i = 0; i < 8; ++i) eoff[i] = ((i + rot) & 7) * 16 + l16;
    }
    FftLaneConst lc;
    load_lane_const(lc, tab.tw_stage, tab.tw_post, l16);
    __syncthreads();

    constexpr int used = 512;
    // spw = streams per warp tile (<= K1F_STREAMS_PER_WARP): small batches spread over more warps
    const int n_tiles = (n + spw - 1) / spw;
    const int gwarp = blockIdx.x * K1F_WARPS + warp, nwarps = gridDim.x * K1F_WARPS;
    uint32_t uses0 = 0, uses1 = 0;                          // completed uses of each staging buffer (mbarrier phase)
    for (int tile = gwarp; tile < n_tiles; tile += nwarps) {
        const int base = tile * spw;
        // ---- bookkeeping: lane i < spw <-> stream base + i
        int cnt = 0;
        {
            const int i = base + lane;
            int sid = -1;
            long long n0 = 0, c0 = 0, ts0 = 0;
            if (lane < spw && i < n) {
                sid = ids ? ids[i] : i;
                n0 = st.n_samples[sid];
                c0 = frames_ready(n0, used, hop);
                cnt = (int)(frames_ready(n0 + chunk, used, hop) - c0);
                ts0 = c0 * hop < n0 ? c0 * hop : n0;
                // LEAN: st_ts0 carries (ring slot of frame c0) << 32 | (c0 * hop - n0) instead; -512 < c0 * hop - n0 <= hop - 512
                if (LEAN) ts0 = ((long long)(int)(c0 % st.ring_rows) << 32) | (long long)(unsigned)(int)(c0 * hop - n0);
            }
            if (lane < spw) {
                ws.st_id[lane] = sid; ws.st_n0[lane] = n0; ws.st_ts0[lane] = ts0; ws.st_cnt[lane] = cnt; ws.st_c0[lane] = c0;
            }
        }
        int incl = cnt;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { int v = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += v; }
        const int nf = __shfl_sync(0xffffffffu, incl, 31);
        for (int j = 0; j < cnt; ++j) { ws.fr_stream[incl - cnt + j] = (short)lane; ws.fr_sub[incl - cnt + j] = (short)j; }
        __syncwarp();

        auto issue = [&](int f0, int stage) {               // lane 0: bulk copies for frames f0, f0+1 of the list
            const int nfr = min(2, nf - f0);
            fence_proxy_async();
            mbar_expect_tx(&ws.bar[stage], 1024u * nfr);
            for (int hf = 0; hf < nfr; ++hf) {
                const int t = ws.fr_stream[f0 + hf];
                const int16_t* chunk_p = pcm + (long long)(base + t) * chunk;
                char* dst = reinterpret_cast<char*>(ws.buf[stage][hf]);
                if (LEAN) {
                    const int sub_off = ws.fr_sub[f0 + hf] * hop;
                    const int rel = (int)(unsigned)(ws.st_ts0[t] & 0xffffffffll) + sub_off;        // first sample of the frame, relative to the chunk
                    if (rel >= 0) {
                        bulk_g2s(dst, chunk_p + rel, 1024u, &ws.bar[stage]);
                    } else {                                  // rel < 0 implies the tail starts at frame c0: offset in the tail = sub * hop
                        const int len0 = min(used, -rel);
                        bulk_g2s(dst, st.tail + (long long)ws.st_id[t] * st.tail_cap + sub_off, 2u * len0, &ws.bar[stage]);
                        if (len0 < used) bulk_g2s(dst + 2 * len0, chunk_p, 2u * (used - len0), &ws.bar[stage]);
                    }
                    continue;
                }
                const long long a0 = (ws.st_c0[t] + ws.fr_sub[f0 + hf]) * hop, n0 = ws.st_n0[t];
                if (a0 >= n0) {
                    bulk_g2s(dst, chunk_p + (a0 - n0), 1024u, &ws.bar[stage]);
                } else {
                    const int len0 = (int)min((long long)used, n0 - a0);
                    bulk_g2s(dst, st.tail + (long long)ws.st_id[t] * st.tail_cap + (a0 - ws.st_ts0[t]), 2u * len0, &ws.bar[stage]);
                    if (len0 < used) bulk_g2s(dst + 2 * len0, chunk_p, 2u * (used - len0), &ws.bar[stage]);
                }
            }
        };
        int stage = 0;
        if (nf > 0 && lane == 0) issue(0, 0);
        for (int f0 = 0; f0 < nf; f0 += 2, stage ^= 1) {
            if (f0 + 2 < nf && lane == 0) issue(f0 + 2, stage ^ 1);
            const bool active = f0 + half < nf;
            float* row = st.ring;
            if (active) {
                const int t = ws.fr_stream[f0 + half];
                if (LEAN) {
                    int slot = (int)(ws.st_ts0[t] >> 32) + ws.fr_sub[f0 + half];                 // fr_sub < ring_rows
                    if (slot >= st.ring_rows) slot -= st.ring_rows;
                    row = st.ring + ((long long)ws.st_id[t] * st.ring_rows + slot) * st.row_stride;
                } else {
                    const long long k = ws.st_c0[t] + ws.fr_sub[f0 + half];
                    row = st.ring + ((long long)ws.st_id[t] * st.ring_rows + (int)(k % st.ring_rows)) * st.row_stride;
                }
            }
            const uint32_t parity = (stage == 0 ? uses0 : uses1) & 1;
            fast_pass(ws, stage, parity, lc, tb, ft, tab, scale, eoff, l16, half, active, row);
            if (stage == 0) ++uses0; else ++uses1;
        }
        // ---- tail + sample counter.  Every old-tail read of this tile is complete (the bulk copies that read it
        // were waited for above).  Lane t < spw derives stream t's copy plan; then the whole warp copies all
        // streams' tails in one flat loop of 16-byte vectors so the loads of different streams overlap.
        int my_nv = 0, my_nold = 0;
        if (lane < spw && ws.st_id[lane] >= 0) {
            const long long n0 = ws.st_n0[lane], n1 = n0 + chunk;
            const long long c1 = ws.st_c0[lane] + ws.st_cnt[lane];
            const long long ts1 = c1 * hop < n1 ? c1 * hop : n1;
            my_nold = ts1 < n0 ? (int)(n0 - ts1) : 0;
            my_nv = ((int)(n1 - ts1) - my_nold) >> 3;
            ws.st_ts0[lane] = ts1 > n0 ? ts1 - n0 : 0;      // reuse: offset of the copied part inside the chunk
            ws.st_cnt[lane] = my_nv | (my_nold << 16);
            st.n_samples[ws.st_id[lane]] = n1;
        }
        const unsigned any_old = __ballot_sync(0xffffffffu, my_nold > 0);
        __syncwarp();
        if (any_old) {                                        // chunk shorter than the FFT window: shift inside the tail first
            for (int t = 0; t < spw; ++t) {
                const int sid = ws.st_id[t];
                if (sid < 0) continue;
                const int n_old = ws.st_cnt[t] >> 16;
                if (n_old == 0) continue;
                const long long n0 = ws.st_n0[t];
                int16_t* tl = st.tail + (long long)sid * st.tail_cap;
                // old tail held [n0 - len0, n0); the part that survives is its last n_old samples
                const long long c0 = frames_ready(n0, used, hop);
                const long long ts0 = c0 * hop < n0 ? c0 * hop : n0;
                const int len0 = (int)(n0 - ts0);
                int4 keep[2];
                const int4* srcv = reinterpret_cast<const int4*>(tl + (len0 - n_old));
                const int nv = n_old >> 3;
#pragma unroll
                for (int j = 0; j < 2; ++j) if (j * 32 + lane < nv) keep[j] = srcv[j * 32 + lane];
                __syncwarp();
#pragma unroll
                for (int j = 0; j < 2; ++j) if (j * 32 + lane < nv) reinterpret_cast<int4*>(tl)[j * 32 + lane] = keep[j];
            }
            __syncwarp();
        }
        // flat loop over (stream, vector) slots, 4 loads in flight per lane before the first store
#pragma unroll 1
        for (int e0 = lane; e0 < spw * 64; e0 += 32 * 4) {
            int4 v[4];
            int4* dst[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int e = e0 + 32 * u;
                dst[u] = nullptr;
                if (e < spw * 64) {
                    const int t = e >> 6, vi = e & 63;
                    const int cn = ws.st_cnt[t];
                    if (ws.st_id[t] >= 0 && vi < (cn & 0xffff)) {
                        v[u] = __ldg(reinterpret_cast<const int4*>(pcm + (long long)(base + t) * chunk + ws.st_ts0[t]) + vi);
                        dst[u] = reinterpret_cast<int4*>(st.tail + (long long)ws.st_id[t] * st.tail_cap + (cn >> 16)) + vi;
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (dst[u] != nullptr) *dst[u] = v[u];
        }
        __syncwarp();
    }
}

// ------------------------------------------------------------------------------------------------
// Stateful tick, pipelined (pb_update / pb_update_vectors on the aligned geometry; k1 mode 2 runs mfcc_fast_stream_kernel<true>
// above instead).  Every frame's arithmetic, the tiling and the frame -> half-warp assignment are mfcc_fast_stream_kernel<true>'s,
// so rows, tails and sample counts are bit-identical to it.  What differs is how the warp waits (DESIGN.md §3 K1):
//   - 5 CTAs of 4 warps per SM instead of 4.  The stage twiddles live in one shared [k1][n2] table per CTA instead of 32
//     registers per lane, the FFT exchange goes through a float scratch one component at a time, the 1 KB input stages are
//     separate from that scratch, and mel16's partials and log-mels live in the input stage the pass has just read.
//   - A tile's stream ids are loaded one tile ahead (their latency hides under the passes) and its sample counts during the
//     previous tile's tail update.
constexpr int K1P_CTAS_PER_SM = 5;
constexpr int K1P_TAIL_INFLIGHT = 4;
constexpr int K1P_MEL_UQ = 1, K1P_MEL_UC = 4;   // mel16's unroll factors
constexpr int K1P_IN_WORDS = 256 + 16;         // 1 KB frame +64 B: the two half-warps' input reads fall in disjoint bank halves
static_assert(K1F_PART + K1_MAX_FILT <= K1P_IN_WORDS, "mel16's part | mel must fit in an input stage");
static_assert(K1F_ZERO_BIN < XCH_ELEMS, "the zero bin must lie in the exchange scratch");

// The mel shape the pipe kernel compiles in (mel16_fixed): the reference's default front end (16 kHz, n_fft 512, 20 filters,
// 13 MFCCs) cuts the spectrum into 41 pieces, three piece blocks of 16 lanes, and sums at most 9 partials into one filter.
// Every other shape runs mel16 with the shape read from the tables.
constexpr int K1P_FIX_NPL = 3, K1P_FIX_MAXC = 9, K1P_FIX_NF = 20, K1P_FIX_NOUT = 13;

struct PipeMelTables {         // mel16_fixed's tables (built by api.cu from ptab / ctab / dct_t); shared-memory copies in the kernel
    const int4* poff;          // [npl][2][32]  lane L's 8 piece entries in L's walk order (see mel16): byte offsets of the bins in P
    const float4* pw;          // [npl][4][32]  the same entries' (w_rise, w_fall), two entries per vector
    const uint4* crow;         // [16 * (n_filt / 16 + 1)]  ctab row j as 16 bytes, padded with the zero slot 128; rows >= n_filt: all 128
    const float4* dct;         // [16][n_filt / 4]  DCT row c (dct_t transposed back), zero for c >= n_out
};

template <int NPL, int NF>
struct PipeMelShape {
    static constexpr int ROWS = 16 * (NF / 16 + 1);                   // filter rows j = l16 + 16 it, slot NF included
    static constexpr size_t BYTES = (size_t)NPL * 6 * 32 * sizeof(int4) + ROWS * sizeof(uint4) + 16 * NF * sizeof(float);
};

// mel16 for a compile-time shape, on the tables above: the same float operations in the same order (the rotated entry walk,
// the r / f / tot chains, the m0 / m1 slot chains, the a0 / a1 DCT chains), with every loop unrolled, the piece entries read
// as 6 vectors per block instead of 8, a filter's slot list as one vector, and the DCT and log-mels 4 filters per load.
// The filter pass has idle lanes when n_filt is not a multiple of 16: lane n_filt - 16 (it) takes log(max(tot, eps)) there,
// which mel16 computes in the DCT for row 0.
template <int NPL, int MAXC, int NF, int NOUT>
__device__ __forceinline__ void mel16_fixed(const float* P, const PipeMelTables& tb, float* part, float* mel, int lane, int l16,
                                            bool active, float* __restrict__ out) {
    static_assert(16 * NPL <= 64 && MAXC <= 16 && NF % 4 == 0 && PipeMelShape<NPL, NF>::ROWS <= K1_MAX_FILT && NOUT <= 16, "shape");
    const char* Pb = reinterpret_cast<const char*>(P);
    float tot = 0.f;
#pragma unroll
    for (int q = 0; q < NPL; ++q) {
        const int4 o0 = tb.poff[(2 * q) * 32 + lane], o1 = tb.poff[(2 * q + 1) * 32 + lane];
        const int off[8] = {o0.x, o0.y, o0.z, o0.w, o1.x, o1.y, o1.z, o1.w};
        float w[16];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float4 v = tb.pw[(4 * q + k) * 32 + lane];
            w[4 * k] = v.x; w[4 * k + 1] = v.y; w[4 * k + 2] = v.z; w[4 * k + 3] = v.w;
        }
        float r = 0.f, f = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float pw = *reinterpret_cast<const float*>(Pb + off[i]);
            tot += pw;
            r = fmaf(w[2 * i], pw, r);
            f = fmaf(w[2 * i + 1], pw, f);
        }
        part[q * 16 + l16] = r;
        part[64 + q * 16 + l16] = f;
    }
#pragma unroll
    for (int d = 8; d >= 1; d >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, d);   // every lane of the half ends with the same sum
    __syncwarp();
#pragma unroll
    for (int it = 0; it <= NF / 16; ++it) {
        const int j = l16 + 16 * it;
        const uint4 row = tb.crow[j];
        const unsigned cw[4] = {row.x, row.y, row.z, row.w};
        float m0 = 0.f, m1 = 0.f;
#pragma unroll
        for (int c = 0; c + 1 < MAXC; c += 2) {
            m0 += part[(cw[c >> 2] >> (8 * (c & 3))) & 255u];
            m1 += part[(cw[(c + 1) >> 2] >> (8 * ((c + 1) & 3))) & 255u];
        }
        if (MAXC & 1) m0 += part[(cw[(MAXC - 1) >> 2] >> (8 * ((MAXC - 1) & 3))) & 255u];
        const float v = (it == NF / 16 && j == NF) ? tot : m0 + m1;
        mel[j] = logf(fmaxf(v, K1_EPS));
    }
    __syncwarp();
    const float4* d = tb.dct + l16 * (NF / 4);
    const float4* m4 = reinterpret_cast<const float4*>(mel);
    float a0 = 0.f, a1 = 0.f;
#pragma unroll
    for (int k = 0; k < NF / 4; ++k) {
        const float4 dv = d[k], mv = m4[k];
        a0 = fmaf(dv.x, mv.x, a0); a1 = fmaf(dv.y, mv.y, a1);
        a0 = fmaf(dv.z, mv.z, a0); a1 = fmaf(dv.w, mv.w, a1);
    }
    const float v = l16 == 0 ? mel[NF] : a0 + a1;
    if (active && l16 < NOUT) out[l16] = v;
    __syncwarp();
}

struct K1PWarp {               // per warp
    int in[2][2][K1P_IN_WORDS];                // [stage][half]: 1 KB input frame (int16 pairs); once read: mel16's part | mel
    float xch[2][XCH_ELEMS];                   // [half]: FFT exchange scratch -> power bins (272 words apart: disjoint bank halves)
    unsigned long long bar[2];
    long long st_n0[K1F_STREAMS_PER_WARP], st_ts0[K1F_STREAMS_PER_WARP], st_c0[K1F_STREAMS_PER_WARP];
    int st_id[K1F_STREAMS_PER_WARP], st_cnt[K1F_STREAMS_PER_WARP];
    int st_vbeg[K1F_STREAMS_PER_WARP];         // tail update: first vector of stream t in the tile's packed vector list
    short fr_stream[K1F_STREAMS_PER_WARP * K1F_MAX_NEW], fr_sub[K1F_STREAMS_PER_WARP * K1F_MAX_NEW];
};
static_assert(sizeof(K1PWarp) % 16 == 0, "every warp's input stages start 16-byte aligned (bulk copy destinations)");

// fast_pass for K1PWarp: the same conversion, FFT and mel stage, with the scratch and the mel stage's arrays placed as above.
// NPL = 0: mel16 on the shape in the tables; its entry offsets are rebuilt from `rot` per pass (the same values) rather than held
// in 8 registers across the tile.  NPL > 0: mel16_fixed.
template <int NPL, int MAXC, int NF, int NOUT>
__device__ __forceinline__ void pipe_pass(K1PWarp& ws, int stage, uint32_t parity, const FftSmemConst& lc, const K1FTab& tb,
                                          const PipeMelTables& pt, const FastTables& ft, const MelTables& t, float scale, int rot,
                                          int lane, int l16, int half, bool active, float* __restrict__ out) {
    mbar_wait(&ws.bar[stage], parity);
    const int* in = ws.in[stage][half];
    cpx z[16];
#pragma unroll
    for (int n1 = 0; n1 < 16; ++n1) {              // int16 pair -> two floats, exactly as fast_pass
        const unsigned v = (active ? (unsigned)in[16 * n1 + l16] : 0u) ^ 0x80008000u;
        z[n1].x = __uint_as_float(__byte_perm(v, 0x4b000000u, 0x7610)) - 8421376.f;
        z[n1].y = __uint_as_float(__byte_perm(v, 0x4b000000u, 0x7632)) - 8421376.f;
    }
    __syncwarp();                                  // all lanes have read the staged samples: the stage becomes mel16's scratch
    float* P = ws.xch[half];
    fft512_power(z, lc, P, P, scale, l16, active); // P aliases the scratch: written after the last scratch read
    float* part = reinterpret_cast<float*>(ws.in[stage][half]);
    if (l16 == 0) { P[K1F_ZERO_BIN] = 0.f; part[128] = 0.f; }
    if constexpr (NPL == 0) {
        int eoff[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) eoff[i] = ((i + rot) & 7) * 16 + l16;
        __syncwarp();
        mel16<K1P_MEL_UQ, K1P_MEL_UC>(P, tb, ft, t, part, part + K1F_PART, eoff, l16, active, out);
    } else {
        __syncwarp();
        mel16_fixed<NPL, MAXC, NF, NOUT>(P, pt, part, part + K1F_PART, lane, l16, active, out);
    }
}

template <int NPL, int MAXC, int NF, int NOUT>
__global__ void __launch_bounds__(K1F_THREADS, K1P_CTAS_PER_SM)
mfcc_pipe_stream_kernel(const int16_t* __restrict__ pcm, const int* __restrict__ ids, int n, int chunk, int hop, int spw,
                        float scale, MelTables tab, FastTables ft, PipeMelTables pmt, StreamState st) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    K1PWarp* wsm = reinterpret_cast<K1PWarp*>(smem_raw);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, l16 = lane & 15, half = lane >> 4;
    K1PWarp& ws = wsm[warp];
    float2* tws = reinterpret_cast<float2*>(smem_raw + K1F_WARPS * sizeof(K1PWarp));
    K1FTab tb{};
    PipeMelTables pt{};
    if constexpr (NPL == 0) {
        tb = load_fast_tables(reinterpret_cast<unsigned char*>(tws + 256), tab, ft);
    } else {                                          // [poff | pw | crow | dct]
        constexpr int NO = NPL * 2 * 32, NW = NPL * 4 * 32, NC = PipeMelShape<NPL, NF>::ROWS, ND = 16 * NF / 4;
        int4* po = reinterpret_cast<int4*>(tws + 256);
        float4* pw = reinterpret_cast<float4*>(po + NO);
        uint4* pc = reinterpret_cast<uint4*>(pw + NW);
        float4* pd = reinterpret_cast<float4*>(pc + NC);
        for (int k = threadIdx.x; k < NO; k += blockDim.x) po[k] = __ldg(pmt.poff + k);
        for (int k = threadIdx.x; k < NW; k += blockDim.x) pw[k] = __ldg(pmt.pw + k);
        for (int k = threadIdx.x; k < NC; k += blockDim.x) pc[k] = __ldg(pmt.crow + k);
        for (int k = threadIdx.x; k < ND; k += blockDim.x) pd[k] = __ldg(pmt.dct + k);
        pt.poff = po; pt.pw = pw; pt.crow = pc; pt.dct = pd;
    }
    for (int k = threadIdx.x; k < 256; k += blockDim.x) tws[k] = tab.tw_stage[(k & 15) * 16 + (k >> 4)];   // [n2][k1] -> [k1][n2]
    if (lane == 0) { mbar_init(&ws.bar[0], 1); mbar_init(&ws.bar[1], 1); fence_mbar_init(); }
    const int rot = ((l16 >> 2) + (half << 2)) & 7;   // rotated walk through a piece: see mel16
    FftSmemConst lc;
    lc.tws = tws + l16;
    {
        const float2 p = tab.tw_post[l16];
        lc.pcr = p.x; lc.psi = p.y;
    }
    __syncthreads();

    constexpr int used = 512;
    const int gwarp = blockIdx.x * K1F_WARPS + warp, nwarps = gridDim.x * K1F_WARPS;
    // lane i < spw: id of stream base + i, -1 past the batch
    auto stream_id = [&](int base) {
        const int i = base + lane;
        return (lane < spw && i < n) ? (ids ? ids[i] : i) : -1;
    };
    int sid = stream_id(gwarp * spw);
    long long n0 = sid >= 0 ? st.n_samples[sid] : 0;
    uint32_t uses0 = 0, uses1 = 0;                          // completed uses of each staging buffer (mbarrier phase)
    for (int base = gwarp * spw; base < n; base += nwarps * spw) {
        const int sid_next = stream_id(base + nwarps * spw);   // in flight across this tile's passes
        // ---- bookkeeping: lane i < spw <-> stream base + i (mfcc_fast_stream_kernel<true>'s encoding of st_ts0)
        int cnt = 0;
        {
            long long c0 = 0, ts0 = 0;
            if (sid >= 0) {
                c0 = frames_ready(n0, used, hop);
                cnt = (int)(frames_ready(n0 + chunk, used, hop) - c0);
                ts0 = ((long long)(int)(c0 % st.ring_rows) << 32) | (long long)(unsigned)(int)(c0 * hop - n0);
            }
            if (lane < spw) {
                ws.st_id[lane] = sid; ws.st_n0[lane] = n0; ws.st_ts0[lane] = ts0; ws.st_cnt[lane] = cnt; ws.st_c0[lane] = c0;
            }
        }
        int incl = cnt;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { int v = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += v; }
        const int nf = __shfl_sync(0xffffffffu, incl, 31);
        for (int j = 0; j < cnt; ++j) { ws.fr_stream[incl - cnt + j] = (short)lane; ws.fr_sub[incl - cnt + j] = (short)j; }
        __syncwarp();

        auto issue = [&](int f0, int stage) {               // lane 0: bulk copies for frames f0, f0+1 of the list
            const int nfr = min(2, nf - f0);
            fence_proxy_async();
            mbar_expect_tx(&ws.bar[stage], 1024u * nfr);
            for (int hf = 0; hf < nfr; ++hf) {
                const int t = ws.fr_stream[f0 + hf];
                const int16_t* chunk_p = pcm + (long long)(base + t) * chunk;
                char* dst = reinterpret_cast<char*>(ws.in[stage][hf]);
                const int sub_off = ws.fr_sub[f0 + hf] * hop;
                const int rel = (int)(unsigned)(ws.st_ts0[t] & 0xffffffffll) + sub_off;        // first sample of the frame, relative to the chunk
                if (rel >= 0) {
                    bulk_g2s(dst, chunk_p + rel, 1024u, &ws.bar[stage]);
                } else {                                  // rel < 0 implies the tail starts at frame c0: offset in the tail = sub * hop
                    const int len0 = min(used, -rel);
                    bulk_g2s(dst, st.tail + (long long)ws.st_id[t] * st.tail_cap + sub_off, 2u * len0, &ws.bar[stage]);
                    if (len0 < used) bulk_g2s(dst + 2 * len0, chunk_p, 2u * (used - len0), &ws.bar[stage]);
                }
            }
        };
        int stage = 0;
        if (nf > 0 && lane == 0) issue(0, 0);
        for (int f0 = 0; f0 < nf; f0 += 2, stage ^= 1) {
            if (f0 + 2 < nf && lane == 0) issue(f0 + 2, stage ^ 1);
            const bool active = f0 + half < nf;
            float* row = st.ring;
            if (active) {
                const int t = ws.fr_stream[f0 + half];
                int slot = (int)(ws.st_ts0[t] >> 32) + ws.fr_sub[f0 + half];                 // fr_sub < ring_rows
                if (slot >= st.ring_rows) slot -= st.ring_rows;
                row = st.ring + ((long long)ws.st_id[t] * st.ring_rows + slot) * st.row_stride;
            }
            const uint32_t parity = (stage == 0 ? uses0 : uses1) & 1;
            pipe_pass<NPL, MAXC, NF, NOUT>(ws, stage, parity, lc, tb, pt, ft, tab, scale, rot, lane, l16, half, active, row);
            if (stage == 0) ++uses0; else ++uses1;
        }
        // the next tile's sample counts: its ids have landed during the passes, the loads overlap the tail update below
        // (stream ids are unique, so no stream of this tile is among them)
        const long long n0_next = sid_next >= 0 ? st.n_samples[sid_next] : 0;
        // ---- tail + sample counter: mfcc_fast_stream_kernel's plan, with the copy over a packed list of the tile's vectors
        int my_nv = 0, my_nold = 0;
        if (lane < spw && ws.st_id[lane] >= 0) {
            const long long n0 = ws.st_n0[lane], n1 = n0 + chunk;
            const long long c1 = ws.st_c0[lane] + ws.st_cnt[lane];
            const long long ts1 = c1 * hop < n1 ? c1 * hop : n1;
            my_nold = ts1 < n0 ? (int)(n0 - ts1) : 0;
            my_nv = ((int)(n1 - ts1) - my_nold) >> 3;
            ws.st_ts0[lane] = ts1 > n0 ? ts1 - n0 : 0;      // reuse: offset of the copied part inside the chunk
            ws.st_cnt[lane] = my_nv | (my_nold << 16);
            st.n_samples[ws.st_id[lane]] = n1;
        }
        int vend = my_nv;                                     // inclusive prefix of the streams' vector counts
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { int v = __shfl_up_sync(0xffffffffu, vend, d); if (lane >= d) vend += v; }
        const int n_vec = __shfl_sync(0xffffffffu, vend, 31);
        if (lane < spw) ws.st_vbeg[lane] = vend - my_nv;
        const unsigned any_old = __ballot_sync(0xffffffffu, my_nold > 0);
        __syncwarp();
        if (any_old) {                                        // chunk shorter than the FFT window: shift inside the tail first
            for (int t = 0; t < spw; ++t) {
                const int sid = ws.st_id[t];
                if (sid < 0) continue;
                const int n_old = ws.st_cnt[t] >> 16;
                if (n_old == 0) continue;
                const long long n0 = ws.st_n0[t];
                int16_t* tl = st.tail + (long long)sid * st.tail_cap;
                // old tail held [n0 - len0, n0); the part that survives is its last n_old samples
                const long long c0 = frames_ready(n0, used, hop);
                const long long ts0 = c0 * hop < n0 ? c0 * hop : n0;
                const int len0 = (int)(n0 - ts0);
                int4 keep[2];
                const int4* srcv = reinterpret_cast<const int4*>(tl + (len0 - n_old));
                const int nv = n_old >> 3;
#pragma unroll
                for (int j = 0; j < 2; ++j) if (j * 32 + lane < nv) keep[j] = srcv[j * 32 + lane];
                __syncwarp();
#pragma unroll
                for (int j = 0; j < 2; ++j) if (j * 32 + lane < nv) reinterpret_cast<int4*>(tl)[j * 32 + lane] = keep[j];
            }
            __syncwarp();
        }
        // flat loop over the tile's n_vec vectors (stream t owns [st_vbeg[t], st_vbeg[t] + its count)), K1P_TAIL_INFLIGHT
        // loads in flight per lane before the first store: ceil(n_vec / 128) round trips, not one per 64 * 2 slots of
        // mfcc_fast_stream_kernel's (stream, vector) grid, most of which are empty
#pragma unroll 1
        for (int e0 = lane; e0 < n_vec; e0 += 32 * K1P_TAIL_INFLIGHT) {
            int4 v[K1P_TAIL_INFLIGHT];
            int4* dst[K1P_TAIL_INFLIGHT];
#pragma unroll
            for (int u = 0; u < K1P_TAIL_INFLIGHT; ++u) {
                const int e = e0 + 32 * u;
                dst[u] = nullptr;
                if (e < n_vec) {
                    int t = 0;                                // the last stream whose first vector is <= e
#pragma unroll
                    for (int b = 8; b >= 1; b >>= 1)
                        if (t + b < spw && ws.st_vbeg[t + b] <= e) t += b;
                    const int vi = e - ws.st_vbeg[t];
                    const int cn = ws.st_cnt[t];
                    v[u] = __ldg(reinterpret_cast<const int4*>(pcm + (long long)(base + t) * chunk + ws.st_ts0[t]) + vi);
                    dst[u] = reinterpret_cast<int4*>(st.tail + (long long)ws.st_id[t] * st.tail_cap + (cn >> 16)) + vi;
                }
            }
#pragma unroll
            for (int u = 0; u < K1P_TAIL_INFLIGHT; ++u)
                if (dst[u] != nullptr) *dst[u] = v[u];
        }
        __syncwarp();
        sid = sid_next;
        n0 = n0_next;
    }
}

}  // namespace pb
