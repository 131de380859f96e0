// corpus_pairs.cuh -- pool models over chosen recordings (pb_score_corpus_pairs): an explicit list of (pool model, recording)
// pairs scanned over the frame buffer K1 builds once per call, as pb_score_corpus_pool does for the full cross product.
//
// Outputs are pair-major: pair p's windows are entries P[p] .. P[p + 1] - 1, P the exclusive prefix over pairs of their
// recordings' window counts.  Pairs are scored in batches of consecutive pairs (at most 2^25 pair-windows each, or one larger
// pair); pw0 holds each batch's own prefix, starting at 0, so every kernel below works in batch-local indices.
//   pairs_windows_kernel  one thread per pair-window of the batch: its start row, copied from its recording's entry of the
//                         window table (a binary search over pw0, as corpus_windows_kernel searches the recordings).
//   pairs_corpus_kernel   one CTA per tile: up to 64 consecutive pair-windows of a run of consecutive pairs on one model, so a
//                         tile may cover several short recordings.  The CTA stages its model from its pool slot and runs
//                         bank_scan in predict mode over the tile's slice of the table: bit-identical to pb_score_corpus_pool.
//   corpus_trigger_kernel corpus.cuh's, with one "recording" per pair and each pair's decoder from its model's slot record.
//   pairs_hits_kernel     one thread per pair-window: decoded conf > hit threshold, compacted with a warp ballot and one
//                         atomicAdd per warp of 32 windows.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "corpus.cuh"
#include "pool.cuh"

namespace pb {

// Pair-windows q0 .. q0 + n - 1 (batch-local, n <= 64) scored by pool slot `slot`.
struct PairTile {
    long long q0;
    int slot;
    int n;
};

__global__ void __launch_bounds__(256) pairs_windows_kernel(const long long* __restrict__ pw0, const int2* __restrict__ pairs, int n_pairs,
                                                            long long n, const long long* __restrict__ win0,
                                                            const long long* __restrict__ starts, long long* __restrict__ starts_p) {
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n) return;
    const int p = corpus_find(pw0, n_pairs, q);
    starts_p[q] = __ldg(starts + __ldg(win0 + __ldg(&pairs[p].y)) + (q - __ldg(pw0 + p)));
}

// bank_scan's view of one tile: one model (position 0), its outputs at the tile's first pair-window.
struct PairsScanP {
    struct W {
        const PoolModel* rec;
        __device__ __forceinline__ const BankModelW& operator[](int) const { return rec->w; }
    } w;
    struct D {
        const PoolModel* rec;
        __device__ __forceinline__ const DecodeParams& operator[](int) const { return rec->dp; }
    } dp;
    struct O {
        float* raw; double* conf;
        __device__ __forceinline__ K2Out operator[](int) const {
            K2Out o{};
            o.raw = raw; o.conf = conf;
            return o;
        }
    } o;
};

// One launch: n_tiles tiles of one activation class.
struct PairsCorpus {
    const uint4* slots;              // the pool's slots
    const PairTile* tiles;           // [n_tiles]
    long long n_tiles;
    const long long* starts;         // [batch pair-windows] the batch's window table
    float* raw;                      // [batch pair-windows] or null
    double* conf;                    // [batch pair-windows] or null
};

// The tile from its linear index over a 2-D grid, as pool_corpus_kernel.  Three CTAs per SM in both forms: at the 128
// registers of four, the run-time activations' form spills 16 B (the tile's own table and output offsets).
template <bool KERAS_ACT>
__global__ void __launch_bounds__(MMA_THREADS, 3)
pairs_corpus_kernel(const __grid_constant__ PairsCorpus c, K2In in) {
    const long long L = (long long)blockIdx.y * gridDim.x + blockIdx.x;
    if (L >= c.n_tiles) return;
    const PairTile t = c.tiles[L];
    PairsScanP P;
    P.w.rec = P.dp.rec = pool_rec(c.slots, t.slot);
    P.o.raw = c.raw ? c.raw + t.q0 : nullptr;
    P.o.conf = c.conf ? c.conf + t.q0 : nullptr;
    in.starts = c.starts + t.q0;
    bank_scan<1, false, KERAS_ACT, PairsScanP>(P, 0, nullptr, 0, in, t.n);
}

// corpus_trigger_kernel's decoders for pairs: "recording" r is pair r of the batch, pool slot pairs[r].x, with the listener's
// refractory count.
struct CorpusPairsDP {
    const uint4* slots;
    const int2* pairs;
    int reset;                       // TriggerDetector(2c bytes)
    __device__ __forceinline__ DecodeParams operator()(int, long long r) const {
        DecodeParams d = pool_rec(slots, __ldg(&pairs[r].x))->dp;
        d.trigger_reset = reset;
        return d;
    }
};

// Hits of one batch: batch-local pair-window q is a hit when decode(raw[q]) > threshold; it is written as q + q_base.
struct PairsHits {
    const float* raw;                // [n]
    const long long* pw0;            // [n_pairs + 1]
    const uint4* slots;
    const int2* pairs;               // [n_pairs] (pool slot, recording)
    long long n, q_base, capacity;
    int n_pairs;
    double threshold;
    int64_t* hits;                   // [capacity] or null (capacity 0)
    unsigned long long* n_hits;      // total, counted past capacity
};

__global__ void __launch_bounds__(256) pairs_hits_kernel(const __grid_constant__ PairsHits H) {
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    bool hit = false;
    if (q < H.n) {
        const int p = corpus_find(H.pw0, H.n_pairs, q);
        const DecodeParams& d = pool_rec(H.slots, __ldg(&H.pairs[p].x))->dp;
        hit = decode_one(__ldg(H.raw + q), d) > H.threshold;       // the comparison train_incremental makes on conf
    }
    const unsigned b = __ballot_sync(0xffffffffu, hit);
    if (b == 0) return;
    unsigned long long at = 0;
    if (lane == 0) at = atomicAdd(H.n_hits, (unsigned long long)__popc(b));
    at = __shfl_sync(0xffffffffu, at, 0);
    const unsigned long long pos = at + (unsigned)__popc(b & ((1u << lane) - 1u));
    if (hit && pos < (unsigned long long)H.capacity) H.hits[pos] = q + H.q_base;
}

}  // namespace pb
