// rows.cuh -- networks given as pb_train weight rows over labelled network inputs (pb_score_rows): precise-test's
// statistics for many networks of up to 128 GRU units without a pool slot or handle weights per network.
//
//   rows_split_kernel     (api.cu, next to upload_wide, which writes the same layout on the host) each network's
//                         gru_wide_kernel fragments from its weight row, and its entry of the group's GruWideW table (bd
//                         included, read from the row on the device)
//   gru_wide_rows_kernel  gru_wide_kernel's tile scan (gru_wide_tile, with its state-update contractions pinned) and W from
//                         the group's table: raw only, inputs in predict mode.  Cross product: grid (tile of 128 inputs,
//                         network of the batch), x fastest, so the CTAs resident at one time share one network's fragments
//                         in L2.  Pairs: one CTA per tile of 128 slots on one network (tile_net), network-major.
//   rows_slots_kernel     pairs: slot s of the batch holds pair slot_pair[s] (or none, -1); its window starts at row rec T
//   rows_scatter_kernel   pairs: raw of each slot back to its pair
//   dataset_stats_kernel  (dataset.cuh, unchanged) the statistics of each batch's raw
//
// gru_wide_kernel's last bit depends on an entry's row within its 16-row block (rows 0-7 and 8-15 take different
// contractions, see gru_wide_tile), so entry r of a cross product sits at row r mod 128 as in pb_predict, and a pair sits in
// a slot of its clip's class ((slot mod 16 < 8) == (rec mod 16 < 8)): its raw equals the cross product's entry however the
// pairs are ordered or cut into batches.  A tile holds up to 64 pairs of each class.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "gru_wide.cuh"

namespace pb {

struct RowsScan {
    const GruWideW* nets;            // cross product: the batch's networks (blockIdx.y); pairs: the group's
    const int* tile_net;             // pairs: [gridDim.x] network of each tile of 128 slots; null: cross product
    float* raw;                      // cross product: [networks of the batch][n]; pairs: [slots]
    long long n;                     // cross product: inputs per network; pairs: slots
};

__global__ void __launch_bounds__(WG_THREADS, 1) gru_wide_rows_kernel(const __grid_constant__ RowsScan S, K2In in) {
    const int net = S.tile_net ? __ldg(S.tile_net + blockIdx.x) : (int)blockIdx.y;
    K2Out o{};
    o.raw = S.tile_net ? S.raw : S.raw + (long long)net * S.n;
    const GruWideW W = S.nets[net];
    gru_wide_tile<false, true>(W, in, [] { return (long long)blockIdx.x * WG_STREAMS; }, S.n, DecodeParams{}, o);
}

__global__ void rows_slots_kernel(const int* __restrict__ slot_pair, const int2* __restrict__ pairs, long long n_slots, int T,
                                  long long* __restrict__ starts) {
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_slots) return;
    const int p = slot_pair[s];
    starts[s] = p >= 0 ? (long long)pairs[p].y * T : 0;
}

__global__ void rows_scatter_kernel(const int* __restrict__ slot_pair, const float* __restrict__ raw_slot, long long n_slots,
                                    float* __restrict__ raw) {
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_slots) return;
    const int p = slot_pair[s];
    if (p >= 0) raw[p] = raw_slot[s];
}

}  // namespace pb
