// pool.cuh -- the model pool (pb_set_pool, pb_pool_load, pb_set_stream_pool, pb_update_pool): up to 2^24 networks of the
// fused family on one handle, each stream scored by at most one of them.
//
// A pool tick runs K1 as every tick does, then:
//   pool_route_kernel   one thread per item: NaN / NaN / 0 for an item whose stream has no pool model; otherwise (item, stream)
//                       goes to its model's list, which starts at list0[m] (the exclusive prefix of the per-model stream counts,
//                       built on the host) in one [max_streams] array.  Lanes with the same model share one atomicAdd.
//   pool_block_kernel   one CTA per block tile: 64 list positions of one model, one weight load per CTA (bank_scan<1>, as
//                       gru_bank_routed_kernel scans a model).
//   pool_warp_kernel    one warp per warp tile: the at most 63 positions past a model's last block tile, as tiles of 16.  The
//                       4 warps of a CTA may score 4 different models, each from its own shared-memory slot.
//   pool_trigger_kernel only once pb_set_stream_pool_trigger has been called: the scans then write raw and conf only, and
//                       this kernel runs each stream's TriggerDetector with its own settings or its model's.
// The tile tables (model, first position) are built on the host whenever assignments or models change, one per tile shape and
// activation class, so a tick reads nothing back.  A tile whose first position is at or past its model's count this tick (a
// tick over a subset of the streams) exits before it loads weights.  Every scan is bank_scan's, with the bank's per-model
// accumulation order: a pool stream scores bit-identically to the same network in a bank.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "gru_bank.cuh"
#include "trigger.cuh"

namespace pb {

// One pool model's device record: its weights (pointers into the pool's fragment array and decoder table) and decoder.
struct PoolModel {
    BankModelW w;
    DecodeParams dp;
};

// A pool slot in the pool-wide slot array: the weights laid out as bank_scan stages them (bfrag, xfrag, bias, wd), then the
// model's record.  One copy replaces both, so a failed load leaves the slot as it was.
constexpr int POOL_FRAG_U4 = BANK_MODEL_SMEM / 16;                  // 888 uint4 = 14 208 B
constexpr int POOL_REC_U4 = (int)((sizeof(PoolModel) + 15) / 16);  // 7 uint4 = 112 B
constexpr int POOL_SLOT_U4 = POOL_FRAG_U4 + POOL_REC_U4;
static_assert(BANK_MODEL_SMEM % 16 == 0, "pool slots are uint4 arrays");

__host__ __device__ __forceinline__ const PoolModel* pool_rec(const uint4* slots, int m) {
    return reinterpret_cast<const PoolModel*>(slots + (size_t)m * POOL_SLOT_U4 + POOL_FRAG_U4);
}

// Everything a pool tick's kernels read and write.  Outputs are [n], indexed by item.
struct PoolTick {
    const int* pool_id;              // [max_streams] model of each stream, -1 = none
    const uint4* slots;              // [max_models][POOL_SLOT_U4]
    int2* lists;                     // [max_streams] (item, stream), model m's list at [list0[m], list0[m + 1])
    unsigned* count;                 // [max_models] list lengths this tick, zeroed before the route
    const unsigned* list0;           // [max_models + 1]
    float* raw;                      // or null
    double* conf;
    uint8_t* fired;                  // or null
    unsigned long long* d_count;     // or null
    int* trig;                       // [max_streams] each stream's pool TriggerDetector.activation
};

// A tick whose ids repeat a stream (outside the contract) could list more items for a model than it has streams: those
// items are not listed (they get NaN / NaN / 0), so no list overruns its range, and every scan stops at its model's range.
__global__ void __launch_bounds__(256) pool_route_kernel(const int* ids, long long n, PoolTick t) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool ok = i < n;
    const int sid = ok ? (ids ? ids[i] : (int)i) : 0;
    const int m = ok ? t.pool_id[sid] : -1;
    if (ok && m < 0) {
        if (t.raw) t.raw[i] = __int_as_float(0x7fc00000);
        t.conf[i] = __longlong_as_double(0x7ff8000000000000LL);
        if (t.fired) t.fired[i] = 0;
    }
    const bool sub = m >= 0;
    const unsigned act = __ballot_sync(0xffffffffu, sub);
    if (!sub) return;
    const int lane = threadIdx.x & 31;
    const unsigned peers = __match_any_sync(act, m);
    const int leader = __ffs(peers) - 1;
    unsigned at = 0;
    if (lane == leader) at = atomicAdd(t.count + m, (unsigned)__popc(peers));
    at = __shfl_sync(peers, at, leader);
    const unsigned pos = t.list0[m] + at + __popc(peers & ((1u << lane) - 1u));
    if (pos < t.list0[m + 1]) {
        t.lists[pos] = make_int2((int)i, sid);
    } else {
        if (t.raw) t.raw[i] = __int_as_float(0x7fc00000);
        t.conf[i] = __longlong_as_double(0x7ff8000000000000LL);
        if (t.fired) t.fired[i] = 0;
    }
}

// Items of model m this tick: its count, at most its list range.
__device__ __forceinline__ long long pool_items(const PoolTick& t, int m) {
    const unsigned c = t.count[m], r = t.list0[m + 1] - t.list0[m];
    return c < r ? c : r;
}

// bank_scan's view of one pool model: P.w[k], P.dp[k] and P.o[k] are that model's whatever k.
struct PoolScanP {
    struct W { const PoolModel* r; __device__ __forceinline__ const BankModelW& operator[](int) const { return r->w; } } w;
    struct D { const PoolModel* r; __device__ __forceinline__ const DecodeParams& operator[](int) const { return r->dp; } } dp;
    struct O { K2Out o; __device__ __forceinline__ const K2Out& operator[](int) const { return o; } } o;
};

__device__ __forceinline__ PoolScanP pool_scan_params(const PoolTick& t, int m) {
    PoolScanP P;
    P.w.r = pool_rec(t.slots, m);
    P.dp.r = P.w.r;
    P.o.o = K2Out{};
    P.o.o.raw = t.raw; P.o.o.conf = t.conf; P.o.o.fired = t.fired; P.o.o.count = t.d_count; P.o.o.trig = t.trig;
    return P;
}

// A pool with per-stream trigger settings (pb_set_stream_pool_trigger): its scans run with trig = fired = d_count = null, so
// epilogue writes raw and conf only, and pool_trigger_kernel updates the detectors afterwards.
struct PoolTrig {
    const int* ids;                  // item -> stream id (null = identity)
    long long n;
    const int* pool_id;              // [max_streams] model of each stream, -1 = none
    const uint4* slots;              // the pool's slots: a stream that follows its model reads the model's DecodeParams
    const double* conf;              // [n] the tick's pool conf
    uint8_t* fired;                  // [n] or null
    unsigned long long* d_count;     // or null
    int* trig;                       // [max_streams] each stream's pool TriggerDetector.activation
    const TrigRec* rec;              // [max_streams] each stream's settings; trigger_reset == 0: the model's own
};

// TriggerDetector.update (runner.py:127-142), one thread per item.  An item whose stream has no pool model gets fired 0 and
// its detector does not move.  Fires are counted with one atomicAdd per warp, as in epilogue.
__global__ void __launch_bounds__(256) pool_trigger_kernel(const __grid_constant__ PoolTrig t) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool ok = i < t.n;
    const int sid = ok ? (t.ids ? t.ids[i] : (int)i) : 0;
    const int m = ok ? t.pool_id[sid] : -1;
    bool fired = false;
    if (m >= 0) {
        const double conf = t.conf[i];
        TrigRec r = t.rec[sid];
        if (r.trigger_reset == 0) {
            const DecodeParams& d = pool_rec(t.slots, m)->dp;
            r.hot_threshold = d.hot_threshold; r.trigger_level = d.trigger_level; r.trigger_reset = d.trigger_reset;
        }
        int a = t.trig[sid];
        const bool hot = conf > r.hot_threshold;
        if (hot || a < 0) {
            a += 1;
            fired = a > r.trigger_level;
            if (fired || (hot && a < 0)) a = r.trigger_reset;
        } else if (a > 0) {
            a -= 1;
        }
        t.trig[sid] = a;
    }
    if (ok && t.fired) t.fired[i] = fired ? 1 : 0;
    if (t.d_count) {
        const unsigned b = __ballot_sync(0xffffffffu, fired);
        if (b && (threadIdx.x & 31) == 0) atomicAdd(t.d_count, (unsigned long long)__popc(b));
    }
}

// tiles[blockIdx.x] = (model, first list position, a multiple of 64).
template <bool KERAS_ACT>
__global__ void __launch_bounds__(MMA_THREADS, 4)
pool_block_kernel(const int2* __restrict__ tiles, const __grid_constant__ PoolTick t, K2In in) {
    const int2 e = tiles[blockIdx.x];
    const long long n = pool_items(t, e.x);
    if (e.y >= n) return;
    bank_scan<1, true, KERAS_ACT, PoolScanP>(pool_scan_params(t, e.x), 0, t.lists + t.list0[e.x], e.y / 64, in, n);
}

// tiles[4 blockIdx.x + warp] = (model, first list position, a multiple of 16), n_tiles of them.  Four CTAs per SM fit in
// shared memory; with run-time activations the scan needs more than the 128 registers that allows (ptxas spills 44 B there),
// so that class runs three.
template <bool KERAS_ACT>
__global__ void __launch_bounds__(MMA_THREADS, KERAS_ACT ? 4 : 3)
pool_warp_kernel(const int2* __restrict__ tiles, long long n_tiles, const __grid_constant__ PoolTick t, K2In in) {
    const long long k = (long long)blockIdx.x * (MMA_THREADS / 32) + (threadIdx.x >> 5);
    if (k >= n_tiles) return;
    const int2 e = tiles[k];
    const long long n = pool_items(t, e.x);
    if (e.y >= n) return;
    bank_scan<1, true, KERAS_ACT, PoolScanP, true>(pool_scan_params(t, e.x), 0, t.lists + t.list0[e.x], e.y / 16, in, n);
}

// Streams sids[j] get model models[j] (-1 = none) and a fresh pool detector.
__global__ void pool_set_kernel(int* pool_id, int* trig, const int* sids, const int* models, long long k) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= k) return;
    pool_id[sids[j]] = models[j];
    trig[sids[j]] = 0;
}

// Every stream on model m gets a fresh pool detector (the model was replaced).
__global__ void pool_rearm_model_kernel(const int* pool_id, int* trig, long long S, int m) {
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s < S && pool_id[s] == m) trig[s] = 0;
}

// Streams ids[i] (or i) get a fresh pool detector (pb_clear).
__global__ void pool_clear_kernel(int* trig, const int* ids, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) trig[ids ? ids[i] : (int)i] = 0;
}

// State records carry the pool detector in header word 14 (pb_stream_state_header.pool_activation).  EXPORT: record i gets
// stream ids[i]'s (or i's) detector; otherwise the stream gets record i's.
template <bool EXPORT>
__global__ void pool_state_kernel(int* trig, const int* ids, long long n, int* recs, long long rec_words) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int sid = ids ? ids[i] : (int)i;
    int* w = recs + i * rec_words + 14;
    if (EXPORT) *w = trig[sid];
    else trig[sid] = *w;
}

}  // namespace pb
