// corpus_pool.cuh -- pool models over a recorded corpus (pb_score_corpus_pool): K1 and the window table once per call, as
// pb_score_corpus builds them, then every requested pool model scans every window of the frame buffer.
//
//   pool_corpus_kernel  one CTA per (window tile of 64, group of NM requested models).  The CTA stages its NM models from
//                       their pool slots (the 14 208 B layout pool_block_kernel stages) and runs bank_scan in predict mode:
//                       each window's rows are read once per step for all NM models, and each model writes raw (and conf
//                       when asked) to its own output row.  Groups are built on the host, per activation class where the
//                       compiled-in Keras activations are used; a last partial group repeats a model of the group at
//                       positions whose output row is -1, which are scanned and written nowhere.
//   corpus_trigger_kernel  corpus.cuh's, with each row's decoder read from its model's pool slot record.
// Every scan is bank_scan's, so a pool row is bit-identical to the same network scored in a bank by pb_score_corpus.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "corpus.cuh"
#include "pool.cuh"

namespace pb {

// bank_scan's view of one group: position j is pool slot e[j].x, written to row e[j].y of raw / conf (-1: nowhere).
struct PoolCorpusScanP {
    struct W {
        const uint4* slots; const int2* e;
        __device__ __forceinline__ const BankModelW& operator[](int j) const { return pool_rec(slots, __ldg(&e[j].x))->w; }
    } w;
    struct D {
        const uint4* slots; const int2* e;
        __device__ __forceinline__ const DecodeParams& operator[](int j) const { return pool_rec(slots, __ldg(&e[j].x))->dp; }
    } dp;
    struct O {
        const int2* e; float* raw; double* conf; long long W;
        __device__ __forceinline__ K2Out operator[](int j) const {
            const long long r = __ldg(&e[j].y);
            K2Out o{};
            if (r >= 0) {
                o.raw = raw ? raw + r * W : nullptr;
                o.conf = conf ? conf + r * W : nullptr;
            }
            return o;
        }
    } o;
};

// One launch: n_groups groups of NM (slot, row) entries over n_tiles tiles of 64 windows.
struct PoolCorpus {
    const uint4* slots;              // the pool's slots
    const int2* groups;              // [n_groups][NM]
    long long n_groups, n_tiles;
    float* raw;                      // [rows][W] or null
    double* conf;                    // [rows][W] or null
    long long W;
    int groups_fast;                 // 1: consecutive CTAs take the groups of one tile; 0: the tiles of one group
};

// The compiled-in Keras activations are used up to NM = 2: above, ptxas interleaves the models' chains and spills, as the
// bank's do (gru_bank.cuh, launch_bank_nm).
constexpr bool pool_corpus_keras(int nm) { return nm <= 2; }

// The CTA's (group, tile) from its linear index over a 2-D grid: gridDim.y <= 65 535 and up to 2^24 models.  NM = 1 with
// the compiled-in activations runs three CTAs per SM: at the 128 registers of four, ptxas spills 8 B in predict mode.
template <int NM, bool KERAS_ACT>
__global__ void __launch_bounds__(MMA_THREADS, NM == 1 ? (KERAS_ACT ? 3 : 4) : 1)
pool_corpus_kernel(const __grid_constant__ PoolCorpus c, K2In in) {
    const long long L = (long long)blockIdx.y * gridDim.x + blockIdx.x;
    if (L >= c.n_groups * c.n_tiles) return;
    const long long g = c.groups_fast ? L % c.n_groups : L / c.n_tiles;
    const long long tile = c.groups_fast ? L / c.n_groups : L % c.n_tiles;
    const int2* e = c.groups + g * NM;
    PoolCorpusScanP P;
    P.w.slots = c.slots; P.w.e = e;
    P.dp.slots = c.slots; P.dp.e = e;
    P.o.e = e; P.o.raw = c.raw; P.o.conf = c.conf; P.o.W = c.W;
    bank_scan<NM, false, KERAS_ACT, PoolCorpusScanP>(P, 0, nullptr, tile, in, c.W);
}

// corpus_trigger_kernel's decoders for pool rows: row m is pool slot ids[m], with the listener's refractory count.
struct CorpusPoolDP {
    const uint4* slots;
    const int* ids;
    int reset;                       // TriggerDetector(2c bytes)
    __device__ __forceinline__ DecodeParams operator()(int m, long long) const {
        DecodeParams d = pool_rec(slots, __ldg(ids + m))->dp;
        d.trigger_reset = reset;
        return d;
    }
};

}  // namespace pb
