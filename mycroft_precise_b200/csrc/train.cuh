// train.cuh -- training of fused-family networks (pb_train, pb_train_loss) and the network input of labelled clips
// (pb_vectorize_clips).  The reference trains with Keras fit (precise/model.py:57-91, scripts/train.py:159-166): GRU with
// reset_after = False, Dense(1, sigmoid), the weighted log loss of precise/functions.py:39-50, the Keras 2.1/2.2 GRU's input
// dropout (implementation 1: one mask per gate z, r, h, [feature_size], fixed over the time steps) and RMSprop.  All
// arithmetic is float32 on the CUDA cores, as Keras trains.
//
//   vectorize_gather_kernel  one thread per (clip, row, feature): the n_features frame rows pb_score_dataset's scan reads
//   train_keys_kernel        the shuffle's sort keys key(s, e, j, 0), with j as the value; cub::DeviceSegmentedSort then
//                            orders each row's entries (a stable sort: ties keep j ascending)
//   train_grad_kernel        one CTA per (row, tile of TR_TILE entries of one batch), one warp per entry at a time, lane =
//                            hidden unit.  The row's weights are staged in shared memory; the forward pass keeps each step's
//                            gate pre-activations and h in the warp's shared state, BPTT runs over the n_features steps,
//                            and the weight gradient is accumulated in the warp's own shared gradient row (a lane writes
//                            only its own columns: no atomics).  The warps' rows are summed in warp order into the
//                            tile's partial gradient, with the tile's loss sum beside it.
//   train_update_kernel      one CTA per row of a batch: the row's partials summed in tile order, then RMSprop (pb_train)
//                            or the gradient written out (pb_train_loss).  The fixed orders make every result independent
//                            of the other rows of the call, of the grouping of rows and of the launch configuration.
//
// Randomness is a function of (seed, epoch, entry, counter): key(s, e, j, c) = mix(mix(mix(mix(s) + e) + j) + c), mix the
// splitmix64 finalizer; dropout keeps feature f of gate g iff float32((key(s, e, j, 1 + 3 f + g) >> 40) 2^-24) >= rate.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pb {

constexpr int TR_STRIDE = 2980;            // floats per weight row: 3 H (F + H + 1) + H + 1 <= 2977 (H = 24, F = 16)
constexpr int TR_MAX_H = 24, TR_MAX_F = 16;
constexpr int TR_WARPS = 4;
constexpr int TR_THREADS = TR_WARPS * 32;
constexpr int TR_TILE = 64;                // entries per gradient CTA (TR_TILE / TR_WARPS per warp)
constexpr int TR_UPDATE_THREADS = 256;

__host__ __device__ __forceinline__ uint64_t tr_mix(uint64_t z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// mix(mix(mix(s) + e) + j): key(s, e, j, c) = tr_mix(tr_entry(s, e, j) + c)
__host__ __device__ __forceinline__ uint64_t tr_entry(uint32_t s, uint64_t e, uint64_t j) {
    return tr_mix(tr_mix(tr_mix((uint64_t)s) + e) + j);
}

__host__ __device__ __forceinline__ int tr_row_size(int F, int H) { return 3 * H * (F + H + 1) + H + 1; }

__global__ void vectorize_gather_kernel(const float* __restrict__ frames, const long long* __restrict__ starts, int row_stride,
                                        int T, int F, long long n, float* __restrict__ out) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n * T * F) return;
    const int f = (int)(e % F);
    const long long q = e / F;
    const int t = (int)(q % T);
    const long long r = q / T;
    out[e] = frames[(starts[r] + t) * row_stride + f];
}

// One trained network: its hidden size, activation codes and seed (pb_train_row).
struct TrainRowDev { int hidden, act, ract; uint32_t seed; };

// Entries i of a tile: position start + i of the row's visiting order (the sorted j's, or j itself without a sort).
struct TrainTile { int row; int base; int start; int count; int batch; };   // batch: entries of the tile's batch (1 / B)
// One row's update after a batch: its tiles [t0, t1) of the launch.
struct TrainStep { int row; int t0, t1; int flags; int n; };   // flags: TR_LAST = the row's last batch of the epoch; n its entries
constexpr int TR_LAST = 1;

struct TrainGrad {
    const float* weights;            // [k][TR_STRIDE]
    const TrainRowDev* rows;         // [k]
    const float* inputs;             // [n_rec][T][F]
    const uint8_t* targets;          // [n_rec]
    const int* ent;                  // group-local entry -> clip
    const int* order;                // group-local visiting order (entry index j within the row), or null: j = position
    const TrainTile* tiles;
    float* part;                     // [tiles][TR_STRIDE]
    double* part_loss;               // [tiles]
    int T, F;
    long long epoch;
    float rate, scale, loss_bias;
};

__device__ __forceinline__ float tr_act(int code, float x) {        // PB_ACT_LINEAR / PB_ACT_TANH
    return code == 0 ? x : tanhf(x);
}
__device__ __forceinline__ float tr_act_grad(int code, float y) {   // from the output
    return code == 0 ? 1.f : 1.f - y * y;
}
__device__ __forceinline__ float tr_ract(int code, float x) {       // PB_RACT_HARD_SIGMOID / PB_RACT_SIGMOID
    return code == 0 ? fminf(fmaxf(fmaf(0.2f, x, 0.5f), 0.f), 1.f) : 1.f / (1.f + expf(-x));
}
// hard_sigmoid passes 0.2 where 0 <= 0.2 x + 0.5 <= 1, bounds included (the gradient of clip_by_value); sigmoid y (1 - y)
__device__ __forceinline__ float tr_ract_grad(int code, float x, float y) {
    if (code == 0) {
        const float s = fmaf(0.2f, x, 0.5f);
        return s >= 0.f && s <= 1.f ? 0.2f : 0.f;
    }
    return y * (1.f - y);
}

// Dynamic shared memory: the row's weights [TR_STRIDE], then per warp its gradient row [TR_STRIDE] and its state
// [T][4][TR_MAX_H] (pre-activations of z, r, h and the h the step started from).
__host__ __device__ constexpr size_t train_smem(int T) {
    return (size_t)(TR_STRIDE + TR_WARPS * (TR_STRIDE + 4 * T * TR_MAX_H)) * sizeof(float);
}

__global__ void __launch_bounds__(TR_THREADS) train_grad_kernel(const __grid_constant__ TrainGrad G) {
    extern __shared__ float sm[];
    const TrainTile tile = G.tiles[blockIdx.x];
    const TrainRowDev rd = G.rows[tile.row];
    const int H = rd.hidden, F = G.F, T = G.T, H3 = 3 * H;
    const int n_w = tr_row_size(F, H);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* w = sm;
    float* g = sm + TR_STRIDE + warp * (TR_STRIDE + 4 * T * TR_MAX_H);
    float* st = g + TR_STRIDE;
    const float* wrow = G.weights + (size_t)tile.row * TR_STRIDE;
    for (int i = threadIdx.x; i < n_w; i += TR_THREADS) w[i] = wrow[i];
    for (int i = lane; i < n_w; i += 32) g[i] = 0.f;
    __syncthreads();
    const float* K = w;
    const float* U = w + F * H3;
    const float* bias = U + H * H3;
    const float* dw = bias + H3;
    const float db = dw[H];
    float* gK = g;
    float* gU = g + F * H3;
    float* gb = gU + H * H3;
    float* gdw = gb + H3;
    const bool on = lane < H;
    const int j = on ? lane : 0;
    const float invB = 1.f / (float)tile.batch;
    double loss = 0.0;
#pragma unroll 1
    for (int i = warp; i < tile.count; i += TR_WARPS) {
        const int pos = tile.start + i;
        const int jj = G.order ? G.order[tile.base + pos] : pos;
        const int rec = G.ent[tile.base + jj];
        const float* x = G.inputs + (size_t)rec * T * F;
        const float y = G.targets[rec] ? 1.f : 0.f;
        // the entry's dropout masks: bit 3 f + g of (m1:m0) keeps feature f for gate g
        unsigned m0 = 0xffffffffu, m1 = 0xffffffffu;
        if (G.rate > 0.f) {
            const uint64_t base = tr_entry(rd.seed, (uint64_t)G.epoch, (uint64_t)jj);
            const float u0 = (float)(unsigned)(tr_mix(base + 1 + lane) >> 40) * 5.9604644775390625e-8f;
            const float u1 = (float)(unsigned)(tr_mix(base + 33 + lane) >> 40) * 5.9604644775390625e-8f;
            m0 = __ballot_sync(0xffffffffu, u0 >= G.rate);
            m1 = __ballot_sync(0xffffffffu, u1 >= G.rate);
        }
        const float sc = G.scale;
        auto mval = [&](int c) -> float { return ((c < 32 ? m0 >> c : m1 >> (c - 32)) & 1u) ? sc : 0.f; };
        // forward
        float h = 0.f;
#pragma unroll 1
        for (int t = 0; t < T; ++t) {
            const float* xt = x + t * F;
            float az = bias[j], ar = bias[H + j], ah = bias[2 * H + j];
            for (int f = 0; f < F; ++f) {
                const float xf = __ldg(xt + f);
                az = fmaf(xf * mval(3 * f), K[f * H3 + j], az);
                ar = fmaf(xf * mval(3 * f + 1), K[f * H3 + H + j], ar);
                ah = fmaf(xf * mval(3 * f + 2), K[f * H3 + 2 * H + j], ah);
            }
            for (int q = 0; q < H; ++q) {
                const float hq = __shfl_sync(0xffffffffu, h, q);
                az = fmaf(hq, U[q * H3 + j], az);
                ar = fmaf(hq, U[q * H3 + H + j], ar);
            }
            const float z = tr_ract(rd.ract, az), r = tr_ract(rd.ract, ar);
            const float rh = on ? r * h : 0.f;
            for (int q = 0; q < H; ++q) ah = fmaf(__shfl_sync(0xffffffffu, rh, q), U[q * H3 + 2 * H + j], ah);
            const float hh = tr_act(rd.act, ah);
            float* s = st + t * 4 * TR_MAX_H;
            if (on) { s[j] = az; s[TR_MAX_H + j] = ar; s[2 * TR_MAX_H + j] = ah; s[3 * TR_MAX_H + j] = h; }
            h = on ? fmaf(z, h, (1.f - z) * hh) : 0.f;
        }
        // Dense + sigmoid + loss
        float lg = on ? h * dw[j] : 0.f;
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) lg += __shfl_xor_sync(0xffffffffu, lg, o);
        const float logit = lg + db;
        const float p = 1.f / (1.f + expf(-logit));
        const float lb = G.loss_bias;
        if (lane == 0)
            loss += (double)(lb * (-(1.f - y) * logf(1.f - p + 1e-7f)) + (1.f - lb) * (-y * logf(p + 1e-7f)));
        const float dp = (lb * (1.f - y) / (1.f - p + 1e-7f) - (1.f - lb) * y / (p + 1e-7f)) * invB;
        const float dlogit = dp * (p * (1.f - p));
        if (on) gdw[j] += dlogit * h;
        if (lane == 0) gdw[H] += dlogit;
        float dh = on ? dlogit * dw[j] : 0.f;
        // BPTT
#pragma unroll 1
        for (int t = T - 1; t >= 0; --t) {
            const float* s = st + t * 4 * TR_MAX_H;
            const float az = on ? s[j] : 0.f, ar = on ? s[TR_MAX_H + j] : 0.f, ah = on ? s[2 * TR_MAX_H + j] : 0.f;
            const float hp = on ? s[3 * TR_MAX_H + j] : 0.f;
            const float z = tr_ract(rd.ract, az), r = tr_ract(rd.ract, ar), hh = tr_act(rd.act, ah);
            const float daz = on ? dh * (hp - hh) * tr_ract_grad(rd.ract, az, z) : 0.f;
            const float dah = on ? dh * (1.f - z) * tr_act_grad(rd.act, hh) : 0.f;
            float dhp = dh * z;
            // lane q: d(r h)_q = sum_j dah_j U[q][2H + j], then the z and r gates' share of dh_(t-1)
            float drh = 0.f;
            for (int c = 0; c < H; ++c) drh = fmaf(__shfl_sync(0xffffffffu, dah, c), on ? U[j * H3 + 2 * H + c] : 0.f, drh);
            const float dar = on ? drh * hp * tr_ract_grad(rd.ract, ar, r) : 0.f;
            dhp = fmaf(drh, r, dhp);
            for (int c = 0; c < H; ++c) {
                const float a = __shfl_sync(0xffffffffu, daz, c), b = __shfl_sync(0xffffffffu, dar, c);
                if (on) dhp = fmaf(a, U[j * H3 + c], fmaf(b, U[j * H3 + H + c], dhp));
            }
            // lane j's columns of the weight gradients
            const float rhp = r * hp;
            for (int q = 0; q < H; ++q) {
                const float hq = __shfl_sync(0xffffffffu, hp, q), rq = __shfl_sync(0xffffffffu, rhp, q);
                if (on) {
                    gU[q * H3 + j] += hq * daz;
                    gU[q * H3 + H + j] += hq * dar;
                    gU[q * H3 + 2 * H + j] += rq * dah;
                }
            }
            if (on) {
                const float* xt = x + t * F;
                for (int f = 0; f < F; ++f) {
                    const float xf = __ldg(xt + f);
                    gK[f * H3 + j] += xf * mval(3 * f) * daz;
                    gK[f * H3 + H + j] += xf * mval(3 * f + 1) * dar;
                    gK[f * H3 + 2 * H + j] += xf * mval(3 * f + 2) * dah;
                }
                gb[j] += daz;
                gb[H + j] += dar;
                gb[2 * H + j] += dah;
            }
            dh = on ? dhp : 0.f;
        }
    }
    __syncthreads();
    // the warps' gradient rows, summed in warp order
    float* out = G.part + (size_t)blockIdx.x * TR_STRIDE;
    const size_t wstride = TR_STRIDE + 4 * (size_t)T * TR_MAX_H;
    for (int i = threadIdx.x; i < n_w; i += TR_THREADS) {
        float a = sm[TR_STRIDE + i];
#pragma unroll
        for (int v = 1; v < TR_WARPS; ++v) a += sm[TR_STRIDE + v * wstride + i];
        out[i] = a;
    }
    __shared__ double s_loss[TR_WARPS];
    if (lane == 0) s_loss[warp] = loss;
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = s_loss[0];
        for (int v = 1; v < TR_WARPS; ++v) a += s_loss[v];
        G.part_loss[blockIdx.x] = a;
    }
}

struct TrainUpdate {
    const TrainStep* steps;
    const TrainRowDev* rows;
    const float* part;
    const double* part_loss;
    float* weights;                  // [k][TR_STRIDE]: RMSprop (pb_train), or null
    float* rms;
    float* grad;                     // [k][TR_STRIDE]: the summed gradient instead (pb_train_loss), or null
    double* loss_acc;                // [k] the epoch's running loss sum
    double* loss;                    // [k][n_loss] or null
    int n_loss, loss_col;
    int F;
    float lr, rho, eps;
};

__global__ void __launch_bounds__(TR_UPDATE_THREADS) train_update_kernel(const __grid_constant__ TrainUpdate P) {
    const TrainStep st = P.steps[blockIdx.x];
    const int n_w = tr_row_size(P.F, P.rows[st.row].hidden);
    const size_t off = (size_t)st.row * TR_STRIDE;
    for (int i = threadIdx.x; i < n_w; i += TR_UPDATE_THREADS) {
        float g = 0.f;
        for (int t = st.t0; t < st.t1; ++t) g += P.part[(size_t)t * TR_STRIDE + i];
        if (P.grad) {
            P.grad[off + i] = g;
        } else if (P.weights) {
            const float a = fmaf(P.rho, P.rms[off + i], (1.f - P.rho) * (g * g));
            P.rms[off + i] = a;
            P.weights[off + i] -= P.lr * g / (sqrtf(a) + P.eps);
        }
    }
    if (threadIdx.x == 0) {
        double a = P.loss_acc[st.row];
        for (int t = st.t0; t < st.t1; ++t) a += P.part_loss[t];
        if (st.flags & TR_LAST) {
            if (P.loss) P.loss[(size_t)st.row * P.n_loss + P.loss_col] = a / (double)st.n;
            a = 0.0;
        }
        P.loss_acc[st.row] = a;
    }
}

__global__ void train_keys_kernel(const TrainRowDev* __restrict__ rows, const int* __restrict__ seg, const int* __restrict__ seg_row,
                                  int n_seg, long long epoch, uint64_t* __restrict__ keys, int* __restrict__ vals) {
    const int s = blockIdx.y;
    if (s >= n_seg) return;
    const int b = seg[s], n = seg[s + 1] - b;
    const uint32_t seed = rows[seg_row[s]].seed;
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
        keys[b + j] = tr_mix(tr_entry(seed, (uint64_t)epoch, (uint64_t)j));
        vals[b + j] = j;
    }
}

}  // namespace pb
