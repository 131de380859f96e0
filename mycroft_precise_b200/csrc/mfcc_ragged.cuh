// mfcc_ragged.cuh -- K1 for ragged ticks on the aligned geometry (n_fft = window crop = 512, hop a multiple of 8): every
// stream brings its own number of samples (pb_update_ragged), so a stream's sample count, its chunk's offset and its length
// have any alignment.  Once a handle has taken a ragged tick, its uniform ticks run here too (implicit offsets i * chunk).
//
// The structure is mfcc_fast_stream_kernel's: a warp owns up to 16 streams, lane i reads stream i's sample count, offset and
// length, and a warp prefix sum builds the list of the frames the tile completes (0..8 per stream and launch; the host runs
// longer chunks as several launches, see RaggedIn).  Each pass transforms two frames with fast_pass (mfcc_fast.cuh) unchanged,
// so a row is bit-identical to the fast kernel's for the same 512 samples.
//
// What differs is the staging.  cp.async.bulk needs 16-byte-aligned addresses and sizes, which an odd offset or sample count
// does not give.  The lanes load the frame themselves instead: lane (half, l16) fetches the 16 sample pairs 16 n1 + l16 of its
// half's frame, with one 32-bit load per pair where both sources (old tail, chunk) are 4-byte aligned and split at an even
// sample, else two 16-bit loads.  Every load addresses one real sample, so nothing outside a stream's part of the packed buffer
// is read.  Before each pass's FFT the warp stages the next pass into the other buffer and lane 0 arrives on that buffer's
// mbarrier, which is what fast_pass waits on.  (Holding the next pass's pairs in registers across the FFT, to hide the load
// latency inside the warp, spills at the 128-register bound; the other warps of the SM hide it instead.)  The tail update
// moves samples one at a time for the same reason as the staging.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "mfcc_fast.cuh"

namespace pb {

struct K1RWarp {               // per warp: the fast kernel's state plus each stream's part of the packed buffer
    K1FWarp f;
    long long st_src[K1F_STREAMS_PER_WARP];
    int st_len[K1F_STREAMS_PER_WARP];
};

__global__ void __launch_bounds__(K1F_THREADS, 4)
mfcc_ragged_stream_kernel(const int16_t* __restrict__ pcm, RaggedIn rg, const int* __restrict__ ids, int n, int hop, int spw,
                          float scale, MelTables tab, FastTables ft, StreamState st) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    K1RWarp* wsm = reinterpret_cast<K1RWarp*>(smem_raw);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, l16 = lane & 15, half = lane >> 4;
    K1RWarp& wr = wsm[warp];
    K1FWarp& ws = wr.f;
    const K1FTab tb = load_fast_tables(smem_raw + K1F_WARPS * sizeof(K1RWarp), tab, ft);
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
    const int n_tiles = (n + spw - 1) / spw;
    const int gwarp = blockIdx.x * K1F_WARPS + warp, nwarps = gridDim.x * K1F_WARPS;
    uint32_t uses0 = 0, uses1 = 0;                          // completed uses of each staging buffer (mbarrier phase)
    for (int tile = gwarp; tile < n_tiles; tile += nwarps) {
        const int base = tile * spw;
        // ---- bookkeeping: lane i < spw <-> stream base + i
        int cnt = 0;
        {
            const int i = base + lane;
            int sid = -1, len = 0;
            long long n0 = 0, c0 = 0, ts0 = 0, src = 0;
            if (lane < spw && i < n) {
                sid = ids ? ids[i] : i;
                ragged_chunk(rg, i, n, src, len);
                n0 = st.n_samples[sid];
                c0 = frames_ready(n0, used, hop);
                cnt = (int)(frames_ready(n0 + len, used, hop) - c0);
                ts0 = c0 * hop < n0 ? c0 * hop : n0;        // first absolute sample held in the tail
            }
            if (lane < spw) {
                ws.st_id[lane] = sid; ws.st_n0[lane] = n0; ws.st_ts0[lane] = ts0; ws.st_cnt[lane] = cnt; ws.st_c0[lane] = c0;
                wr.st_src[lane] = src; wr.st_len[lane] = len;
            }
        }
        int incl = cnt;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { int v = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += v; }
        const int nf = __shfl_sync(0xffffffffu, incl, 31);
        for (int j = 0; j < cnt; ++j) { ws.fr_stream[incl - cnt + j] = (short)lane; ws.fr_sub[incl - cnt + j] = (short)j; }
        __syncwarp();

        // this lane's 16 sample pairs of list frame f -> its half's staging buffer: samples [0, len0) from p0 (the old tail, or
        // the chunk when the frame starts inside it), the rest from p1 (the chunk)
        auto stage_frame = [&](int f, int stage) {
            const int t = ws.fr_stream[f];
            const long long a0 = (ws.st_c0[t] + ws.fr_sub[f]) * hop, n0 = ws.st_n0[t];
            const int16_t* p1 = pcm + wr.st_src[t];
            const int16_t* p0;
            int len0;
            if (a0 >= n0) {
                p0 = p1 + (a0 - n0); p1 = p0; len0 = used;
            } else {
                len0 = (int)min((long long)used, n0 - a0);
                p0 = st.tail + (long long)ws.st_id[t] * st.tail_cap + (a0 - ws.st_ts0[t]);
            }
            uint32_t* dst = reinterpret_cast<uint32_t*>(ws.buf[stage][half]);
            if (((((uintptr_t)p0 | (uintptr_t)p1) & 3) | (len0 & 1)) == 0) {
#pragma unroll
                for (int n1 = 0; n1 < 16; ++n1) {
                    const int s = 2 * (16 * n1 + l16);
                    dst[16 * n1 + l16] = __ldg(reinterpret_cast<const uint32_t*>(s < len0 ? p0 + s : p1 + (s - len0)));
                }
            } else {
#pragma unroll 8
                for (int n1 = 0; n1 < 16; ++n1) {
                    const int s = 2 * (16 * n1 + l16);
                    const uint32_t lo = (uint16_t)__ldg(s < len0 ? p0 + s : p1 + (s - len0));
                    const uint32_t hi = (uint16_t)__ldg(s + 1 < len0 ? p0 + s + 1 : p1 + (s + 1 - len0));
                    dst[16 * n1 + l16] = lo | (hi << 16);
                }
            }
        };
        auto stage_pass = [&](int f0, int stage) {      // all lanes: frames f0, f0 + 1 of the list, then lane 0 arrives
            if (f0 + half < nf) stage_frame(f0 + half, stage);
            __syncwarp();
            if (lane == 0) mbar_arrive(&ws.bar[stage]);
        };
        int stage = 0;
        if (nf > 0) stage_pass(0, 0);
        for (int f0 = 0; f0 < nf; f0 += 2, stage ^= 1) {
            if (f0 + 2 < nf) stage_pass(f0 + 2, stage ^ 1);   // the next pass's frames into the other buffer (its last pass is done)
            const bool active = f0 + half < nf;
            float* row = st.ring;
            if (active) {
                const int t = ws.fr_stream[f0 + half];
                const long long k = ws.st_c0[t] + ws.fr_sub[f0 + half];
                row = st.ring + ((long long)ws.st_id[t] * st.ring_rows + (int)(k % st.ring_rows)) * st.row_stride;
            }
            const uint32_t parity = (stage == 0 ? uses0 : uses1) & 1;
            fast_pass(ws, stage, parity, lc, tb, ft, tab, scale, eoff, l16, half, active, row);
            if (stage == 0) ++uses0; else ++uses1;
        }
        // ---- tail + sample counter.  Every old-tail read of this tile is complete (the fetched pairs were stored above).
        // Lane t < spw derives stream t's plan: keep the last n_old samples of the old tail, append m samples of the chunk.
        int my_nold = 0;
        if (lane < spw && ws.st_id[lane] >= 0) {
            const long long n0 = ws.st_n0[lane], n1 = n0 + wr.st_len[lane];
            const long long c1 = ws.st_c0[lane] + ws.st_cnt[lane];
            const long long ts1 = c1 * hop < n1 ? c1 * hop : n1;
            my_nold = ts1 < n0 ? (int)(n0 - ts1) : 0;
            const int m = (int)(n1 - ts1) - my_nold;               // < 512: frame c1 is not complete
            ws.st_c0[lane] = ts1 - ws.st_ts0[lane];                // reuse: where the kept samples start in the old tail
            wr.st_src[lane] += ts1 > n0 ? ts1 - n0 : 0;            // reuse: first chunk sample that goes to the tail
            ws.st_cnt[lane] = m | (my_nold << 16);
            st.n_samples[ws.st_id[lane]] = n1;
        }
        const unsigned any_old = __ballot_sync(0xffffffffu, my_nold > 0);
        __syncwarp();
        if (any_old) {                                        // chunk shorter than the FFT window: shift inside the tail first
            for (int t = 0; t < spw; ++t) {
                const int sid = ws.st_id[t];
                const int n_old = sid >= 0 ? ws.st_cnt[t] >> 16 : 0;
                if (n_old == 0) continue;
                int16_t* tl = st.tail + (long long)sid * st.tail_cap;
                const int16_t* from = tl + ws.st_c0[t];
                int16_t keep[16];                                 // n_old < 512 = 16 * 32
#pragma unroll
                for (int j = 0; j < 16; ++j) if (j * 32 + lane < n_old) keep[j] = from[j * 32 + lane];
                __syncwarp();
#pragma unroll
                for (int j = 0; j < 16; ++j) if (j * 32 + lane < n_old) tl[j * 32 + lane] = keep[j];
            }
            __syncwarp();
        }
        // chunk samples -> tail, 4 loads in flight per lane before the first store
        for (int t = 0; t < spw; ++t) {
            const int sid = ws.st_id[t];
            if (sid < 0) continue;
            const int cn = ws.st_cnt[t], m = cn & 0xffff;
            const int16_t* from = pcm + wr.st_src[t];
            int16_t* to = st.tail + (long long)sid * st.tail_cap + (cn >> 16);
#pragma unroll 1
            for (int k0 = lane; k0 < m; k0 += 32 * 4) {
                int16_t x[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) if (k0 + 32 * u < m) x[u] = __ldg(from + k0 + 32 * u);
#pragma unroll
                for (int u = 0; u < 4; ++u) if (k0 + 32 * u < m) to[k0 + 32 * u] = x[u];
            }
        }
        __syncwarp();
    }
}

}  // namespace pb
