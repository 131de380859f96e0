// trigger.cuh -- per-stream TriggerDetector settings (pb_set_stream_trigger).
//
// A model whose streams carry their own (sensitivity, trigger_level, chunk_size) is scanned with K2Out.trig = fired = count =
// null, so epilogue writes raw and conf only; trigger_kernel then runs TriggerDetector.update (runner/precise_runner/
// runner.py:127-142) for every (item, model) pair of the tick from the pair's conf and the stream's record.  The scan kernels
// keep their code, and conf is the same either way, so fired equals the fused epilogue's bit for bit on equal settings.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/precise_b200.h"

namespace pb {

// One stream's TriggerDetector of one model: 16 B.
struct TrigRec {
    double hot_threshold;            // 1.0 - sensitivity (runner.py:130), computed on the host in double
    int trigger_level;
    int trigger_reset;               // -(8*2048) // chunk_bytes  (python floor division)
};

// The flagged models of one tick.  Outputs are the model's rows ([n] each, already offset into the [M][n] layout).
struct TrigTick {
    const double* conf[PB_MAX_MODELS];
    uint8_t* fired[PB_MAX_MODELS];               // or null
    unsigned long long* count[PB_MAX_MODELS];    // or null
    int* trig[PB_MAX_MODELS];                    // [max_streams] TriggerDetector.activation
    const TrigRec* rec[PB_MAX_MODELS];           // [max_streams]
    unsigned route_bit[PB_MAX_MODELS];           // the model's bit of route[sid]
    const uint8_t* route;                        // per-stream model masks, or null: every pair is scored
    const int* ids;                              // item -> stream id (null = identity)
    long long n;
};

// blockIdx.y = flagged model k, one thread per item.  A pair whose stream lacks the model's bit is skipped: route_kernel has
// written its NaN / NaN / 0, and its detector does not move.  Fires are counted with one atomicAdd per warp, as in epilogue.
__global__ void __launch_bounds__(256) trigger_kernel(const __grid_constant__ TrigTick t) {
    const int k = blockIdx.y;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    bool valid = i < t.n;
    const int sid = valid ? (t.ids ? t.ids[i] : (int)i) : 0;
    if (valid && t.route && !(t.route[sid] & t.route_bit[k])) valid = false;
    bool fired = false;
    if (valid) {
        const double conf = t.conf[k][i];
        const TrigRec r = t.rec[k][sid];
        int a = t.trig[k][sid];
        const bool hot = conf > r.hot_threshold;
        if (hot || a < 0) {
            a += 1;
            fired = a > r.trigger_level;
            if (fired || (hot && a < 0)) a = r.trigger_reset;
        } else if (a > 0) {
            a -= 1;
        }
        t.trig[k][sid] = a;
        if (t.fired[k]) t.fired[k][i] = fired ? 1 : 0;
    }
    if (t.count[k]) {
        const unsigned m = __ballot_sync(0xffffffffu, fired);
        if (m && (threadIdx.x & 31) == 0) atomicAdd(t.count[k], (unsigned long long)__popc(m));
    }
}

// Stream sids[j] of one model gets record recs[j] and a fresh detector (its values changed).
__global__ void set_trigger_kernel(TrigRec* rec, int* trig, const int* sids, const TrigRec* recs, long long k) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= k) return;
    const int sid = sids[j];
    rec[sid] = recs[j];
    trig[sid] = 0;
}

}  // namespace pb
