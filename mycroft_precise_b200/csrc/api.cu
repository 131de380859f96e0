// api.cu -- C ABI of libprecise_b200.so (see include/precise_b200.h for the contract and the
// reference interface each entry point replaces).  Host side: table construction (float64, then
// rounded once), per-stream state allocation, launch configuration, the pinned/pipelined host
// entry point and CUDA-event profiling.  No CPU compute path exists here by design.
#include <cuda_runtime.h>
#include <math.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <cuda_fp16.h>
#include <limits>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <utility>
#include <vector>

#include "../../include/precise_b200.h"
#include "gru_kernels.cuh"
#include "gru_bank.cuh"
#include "gru_wide.cuh"
#include "mfcc_kernels.cuh"
#include "mfcc_fast.cuh"
#include "mfcc_ragged.cuh"
#include "mfcc_tc.cuh"
#include "mfcc_tc3.cuh"
#include "mfcc_mma.cuh"
#include "trigger.cuh"
#include "stream_state.cuh"
#include "history.cuh"
#include "corpus.cuh"
#include "corpus_pool.cuh"
#include "corpus_pairs.cuh"
#include "dataset.cuh"
#include "pool.cuh"
#include "train.cuh"

#include <cub/device/device_segmented_sort.cuh>

using namespace pb;

// ------------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";

static int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

#define CK(call)                                                                                  \
    do {                                                                                          \
        cudaError_t e_ = (call);                                                                  \
        if (e_ != cudaSuccess)                                                                    \
            return fail(PB_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

constexpr int N_PROFILE_SLOTS = 4;
constexpr int PROFILE_POOL = 2048;
constexpr int K2_WARP_PATH_MAX = 8192;       // streams: below this the warp-per-stream GRU kernel wins (latency-bound regime)
constexpr int64_t HOST_ZERO_COPY_MAX = 64;  // streams: at or below this pb_update_host works in place on pinned host buffers
constexpr int HOST_PIPE = 3;                 // internal streams of pb_update_host
constexpr int64_t HOST_SUB_BATCH = 16384;    // streams per pipelined sub-batch (32 MiB of PCM at 1024 samples)

struct ProfSlot {
    std::vector<cudaEvent_t> ev;   // pairs
    int used = 0;
    double ms = 0.0;
    uint64_t launches = 0;
};

// Device memory of `n` elements of T, freed when the owner goes away.  cudaFree acts on the current device, so every entry
// point that can destroy or replace one (pb_create on failure, pb_destroy, pb_load_weights, pb_add_model) sets the handle's
// device first.
template <typename T>
class DevArray {
public:
    DevArray() = default;
    DevArray(DevArray&& o) noexcept : p_(o.p_), n_(o.n_) { o.p_ = nullptr; o.n_ = 0; }
    DevArray& operator=(DevArray&& o) noexcept { std::swap(p_, o.p_); std::swap(n_, o.n_); return *this; }
    DevArray(const DevArray&) = delete;
    DevArray& operator=(const DevArray&) = delete;
    ~DevArray() { if (p_) cudaFree(p_); }

    // Uninitialised memory.  alloc and upload replace (and free) what the array held only when they succeed.
    cudaError_t alloc(size_t n) {
        T* p = nullptr;
        const cudaError_t e = cudaMalloc((void**)&p, std::max<size_t>(n, 1) * sizeof(T));
        if (e != cudaSuccess) return e;
        DevArray fresh;
        fresh.p_ = p; fresh.n_ = n;
        *this = std::move(fresh);
        return cudaSuccess;
    }
    cudaError_t upload(const std::vector<T>& v) {
        DevArray fresh;
        cudaError_t e = fresh.alloc(v.size());
        if (e == cudaSuccess && !v.empty()) e = cudaMemcpy(fresh.p_, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice);
        if (e == cudaSuccess) *this = std::move(fresh);
        return e;
    }
    T* get() const { return p_; }
    size_t size() const { return n_; }

private:
    T* p_ = nullptr;
    size_t n_ = 0;
};

// One network's weights in every layout a kernel reads (load_weights builds them all at once; they never change after).
struct NetWeights {
    bool small_path = false;         // the default network (H = 20, F = 13, linear / hard_sigmoid): gru_warp / gru_small / gru_bank<1>
    GruSmallW<20, 13> w_small;       // ... its weights as a kernel parameter
    DevArray<float> wcat, bias, wd;  // gru_tiled_kernel: [W; U], bias, dense weights (gru_wide_kernel reads wd as well)
    float bd = 0.f;
    DevArray<uint4> bfrag16;         // fused family (gru_bank_kernel): recurrent weights as fp16 hi / lo fragments
    DevArray<uint4> xfrag16;         // ... and the input weights
    DevArray<float> mma_bias, mma_wd;
    bool wide_ok = false;            // gru_wide_kernel covers the network (H <= 128, F <= 40)
    int wg_fp = 0, wg_hp = 0;
    DevArray<uint4> wg_b1, wg_b2; DevArray<float> wg_bias;
};

// A stream's TriggerDetector arguments as pb_set_stream_trigger took them (the host mirror of a TrigRec).
struct StreamTrig {
    double sensitivity;
    int32_t trigger_level;
    int32_t chunk_bytes;
};

// One model of a handle's bank: its network, ThresholdDecoder table, TriggerDetector state and weights.  It reads the
// handle's MFCC ring; the front-end fields of its cfg equal the handle's.
struct Network {
    pb_config cfg;                   // network (hidden, activations), decoder and trigger fields
    std::vector<double> cd;          // decoder table (build_cdf, or pb_set_cdf / pb_add_model's cd)
    int min_out = 0, max_out = 0;
    DevArray<double> d_cd;
    DevArray<int> trig;              // [max_streams] TriggerDetector.activation
    int gru_mode = 0;                // 0 = auto, 1 = force CUDA-core kernel, 2 = force tensor-core kernel (pb_debug_gru_mode, slot 0)
    std::unique_ptr<NetWeights> w;   // null until weights are loaded
    // per-stream TriggerDetector settings (pb_set_stream_trigger); a model that never gets them keeps trig_set = false and
    // its scan updates the trigger in epilogue, as before
    bool trig_set = false;           // sticky, set by the first pb_set_stream_trigger on this slot
    std::vector<StreamTrig> trig_host;  // [max_streams] the settings as set (defaults until then)
    DevArray<TrigRec> trig_rec;      // [max_streams] their records, read by trigger_kernel
};

// A handle: the MFCC front end (tables, per-stream sample count, tail and ring), the host pipeline and the profiler, shared
// by the models[] it scores.  models[0] is the handle's own network (pb_load_weights), 1.. come from pb_add_model.
struct pb_handle {
    pb_config cfg;                   // the front end; its network fields are models[0]'s
    int sm_count = 132;
    // derived
    int used = 0, n_bins = 0, n_out = 0, feat = 0, ring_rows = 0, row_stride = 0, tail_cap = 0, max_new = 0;
    int rel_window = 0;              // samples before frame 0 is released: window_samples (sonopy), window_samples + hop_samples (speechpy drops the last complete frame)
    size_t k1_batch_smem = 0, k1_stream_smem = 0, k1_fast_smem = 0, k1_pipe_smem = 0, k1_ragged_smem = 0;
    bool ragged = false;             // set by the first pb_update_ragged: n_samples may no longer be a multiple of 8, so every later tick's
                                     // K1 runs launch_ragged_mfcc (the aligned-only kernels would mis-stage it)
    bool force_generic = false;      // tests: exercise the generic kernels on the aligned geometry
    int k1_mode = 0;                 // 0 = default (the pipelined FFT kernel where the geometry allows it), 2 = always the FFT kernel it replaced, 3 = FFT kernel with the original 64-bit set-up, 4 / 5 / 6 = the mma.sync DFT tick (mfcc_mma.cuh): stage 1 on the CUDA cores / on the tensor cores / the latter with a shuffle epilogue
    bool mma_ok = false;             // geometry mfcc_mma_kernel covers (n_fft = frame = 512, hop >= 512, chunk >= hop, MFCC vectorizer)
    DevArray<uint2> d_mm_b1, d_mm_b2; DevArray<float2> d_mm_tw;
    DevArray<MmRec> d_mm_recs; DevArray<unsigned int> d_mm_counters;
    int mm_parity = 0;               // which of the two frame counters the next tick's plan kernel fills
    bool fast_ok = false;            // aligned geometry: warp-autonomous kernels (mfcc_fast.cuh)
    int npl = 0, maxc = 0, nol = 0;
    DevArray<float4> d_ptab;
    DevArray<unsigned char> d_ctab;
    DevArray<float> d_dct_t;
    std::vector<double> fb;          // [n_filt][n_bins] (pb_get_filterbank)
    // device tables
    DevArray<float> d_wrise, d_wfall, d_dct;
    DevArray<int> d_grid;
    DevArray<float2> d_tw_stage, d_tw_post, d_tw_any;
    // per-stream state (stream_state)
    DevArray<long long> d_n_samples;
    DevArray<int16_t> d_tail;
    DevArray<float> d_ring;
    std::vector<Network> models;
    // per-stream model subscriptions (pb_set_stream_models); a handle that never sets them keeps routed = false and none of this
    bool routed = false;             // sticky, set by the first pb_set_stream_models
    std::vector<uint8_t> route_mask; // host mirror of d_route
    int64_t subs[PB_MAX_MODELS] = {};  // streams with bit m set, for all PB_MAX_MODELS bits (a model added later finds its count)
    DevArray<uint8_t> d_route;       // [max_streams] masks, bit m = bank slot m scores the stream
    DevArray<int2> d_route_list;     // [PB_MAX_MODELS][max_streams] route_kernel's (item, stream) lists: scratch of bank ticks
    DevArray<unsigned> d_route_count;  // [PB_MAX_MODELS] their lengths
    cudaEvent_t route_ev = nullptr;  // recorded after each routed bank tick; the next one waits on it before reusing the scratch
    // stream audio history (pb_set_history); a handle without a pool keeps history = false and launches none of this
    bool history = false;            // a pool exists
    int64_t hist_samples = 0;        // history_samples as set
    int hist_cap = 0;                // row length: hist_samples rounded up to a multiple of 8
    int hist_rows = 0;               // max_rows
    DevArray<int16_t> d_hist;        // [hist_rows][hist_cap] the pool
    DevArray<int> d_hist_row;        // [max_streams] row of each stream, -1 = off
    DevArray<long long> d_hist_start;  // [max_streams] history start
    std::vector<int> hist_row;       // host mirror of d_hist_row
    std::vector<int> hist_free;      // rows no stream owns
    // recorded corpora (pb_score_corpus): a workspace that grows on demand and never shrinks
    DevArray<float> d_cw_rows;       // the frame buffer (corpus.cuh)
    DevArray<CorpusPair> d_cw_pairs; // K1's pair list
    DevArray<long long> d_cw_starts; // [windows] first row of each window
    DevArray<long long> d_cw_win0;   // [n_rec + 1] window prefix
    DevArray<long long> d_cw_frow;   // [n_rec] row of each recording's frame 0
    DevArray<CorpusRec> d_cw_recs;   // [n_rec + 1] recordings in pair-list order
    cudaEvent_t corpus_ev = nullptr; // recorded after each corpus call; the next one waits on it before reusing the workspace
    DevArray<int2> d_cp_groups;      // pb_score_corpus_pool: the scan's model groups, (pool slot, output row) entries
    DevArray<int> d_cp_ids;          // ... the requested pool slots, one per output row
    DevArray<float> d_cp_raw;        // ... raw of one batch of rows when the caller passes no d_raw (at most CORPUS_POOL_RAW_CAP bytes)
    int64_t corpus_pool_rows = 0;    // pb_debug_corpus_pool_rows: at most this many rows per batch (0 = the cap's)
    int corpus_pool_nm = 0;          // pb_debug_corpus_pool_scan: models per group (0 = CORPUS_POOL_NM)
    int corpus_pool_order = -1;      // ... grid order (-1 = CORPUS_POOL_GROUPS_FAST)
    DevArray<int2> d_pp_pairs;       // pb_score_corpus_pairs: [n_pairs] (pool slot, recording); raw of a batch goes to d_cp_raw
    DevArray<long long> d_pp_pw0;    // ... each batch's pair-window prefix, batch b's at [p0 + b, p1 + b]
    DevArray<long long> d_pp_starts; // ... [batch pair-windows] the batch's window table
    DevArray<PairTile> d_pp_tiles;   // ... the batch's scan tiles, one activation class after the other
    DevArray<float> d_ds_thr;        // pb_score_dataset: the histogram's float32 thresholds
    DevArray<uint8_t> d_ds_targets;  // ... [n_rec] the recordings' labels
    DevArray<uint8_t> d_tr_ws;       // pb_train / pb_train_loss: one arena, carved per call (at most TRAIN_WS_CAP bytes per group)
    int64_t corpus_pairs_batch = 0;  // pb_debug_corpus_pairs_batch: at most this many pair-windows per batch (0 = CORPUS_PAIRS_BATCH)
    // model pool (pb_set_pool, pool.cuh); a handle without one keeps pool = false and launches none of this
    bool pool = false;               // a pool exists
    int32_t pool_models = 0;         // max_models
    DevArray<uint4> d_pool_slots;    // [max_models][POOL_SLOT_U4] each slot's weights as bank_scan stages them, then its record
    DevArray<unsigned> d_pool_count; // [max_models] list lengths of the current tick (scratch)
    DevArray<unsigned> d_pool_list0; // [max_models + 1] first list position of each model: exclusive prefix of pool_subs
    DevArray<int> d_pool_id;         // [max_streams] model of each stream, -1 = none
    DevArray<int> d_pool_trig;       // [max_streams] each stream's pool TriggerDetector.activation
    DevArray<int2> d_pool_list;      // [max_streams] pool_route_kernel's (item, stream) lists (scratch)
    DevArray<int2> d_pool_tiles[2][2];   // [block, warp][run-time activations, Keras's defaults] (model, first position)
    int64_t pool_tiles[2][2] = {};   // ... and their lengths
    std::vector<int> pool_id;        // host mirror of d_pool_id
    std::vector<int64_t> pool_subs;  // [max_models] streams on each model
    std::vector<uint8_t> pool_keras; // [max_models] 1: the slot's network has Keras's default activations
    struct PoolCd { DevArray<double> d; int64_t refs = 0; };
    std::map<std::string, PoolCd> pool_cd;                  // decoder tables, shared by content (the table's bytes)
    std::vector<std::map<std::string, PoolCd>::iterator> pool_cd_of;  // [max_models] each slot's table; pool_cd.end() = empty slot
    cudaEvent_t pool_ev = nullptr;   // recorded after each pool tick; the next one waits on it before reusing the scratch
    bool pool_warp_only = false;     // pb_debug_pool_tiles: every position in warp tiles
    // per-stream pool TriggerDetector settings (pb_set_stream_pool_trigger); a pool that never gets them keeps pool_trig_set =
    // false and its scans update the trigger in epilogue
    bool pool_trig_set = false;      // sticky until the pool is replaced or freed
    std::vector<StreamTrig> pool_trig_host;  // [max_streams] the settings as set; (NaN, 0, 0) = the stream's model's own
    DevArray<TrigRec> d_pool_trig_rec;       // [max_streams] their records (trigger_reset 0 = the model's own), read by pool_trigger_kernel
    // host pipeline
    cudaStream_t pipe[HOST_PIPE] = {nullptr, nullptr, nullptr};
    cudaEvent_t pipe_ev[HOST_PIPE] = {nullptr, nullptr, nullptr};
    DevArray<int16_t> d_stage_pcm[HOST_PIPE];
    DevArray<int> d_stage_ids[HOST_PIPE];
    DevArray<float> d_stage_raw[HOST_PIPE];
    DevArray<double> d_stage_conf[HOST_PIPE];
    DevArray<uint8_t> d_stage_fired[HOST_PIPE];
    DevArray<unsigned long long> d_count;
    unsigned long long* h_count_pinned = nullptr;
    // profiling
    bool profiling = false;
    ProfSlot prof[N_PROFILE_SLOTS];

    pb_handle() = default;
    pb_handle(const pb_handle&) = delete;
    pb_handle& operator=(const pb_handle&) = delete;
    ~pb_handle() {
        if (h_count_pinned) cudaFreeHost(h_count_pinned);
        for (int i = 0; i < HOST_PIPE; ++i) {
            if (pipe[i]) cudaStreamDestroy(pipe[i]);
            if (pipe_ev[i]) cudaEventDestroy(pipe_ev[i]);
        }
        for (auto& p : prof)
            for (auto e : p.ev) cudaEventDestroy(e);
        if (route_ev) cudaEventDestroy(route_ev);
        if (corpus_ev) cudaEventDestroy(corpus_ev);
        if (pool_ev) cudaEventDestroy(pool_ev);
    }
};

// ------------------------------------------------------------------------------------------------
// table construction (host, float64), restating sonopy.filterbanks as the reference calls it
// (precise/vectorization.py:36-39): grid up to sample_rate, int() truncation, duplicate bins pushed
// forward, np.linspace(endpoint=False) edge weights.
struct MelHost {
    std::vector<int> grid;            // [n_filt + 2] corner bins
    std::vector<float> wrise, wfall;  // [n_bins] weight of a bin on the rising / falling edge of its triangle
    std::vector<double> fb;           // [n_filt][n_bins]
};

static int build_mel(const pb_config& c, int n_bins, MelHost& mel) {
    const int nb = n_bins, nf = c.n_filt;
    const double top = 1127.0 * log(1.0 + (double)c.sample_rate / 700.0);
    std::vector<int>& grid = mel.grid;
    std::vector<double>& fb = mel.fb;
    grid.assign(nf + 2, 0);
    long long shift = 0, prev = -1;
    if (c.vectorizer == PB_VEC_SPEECHPY_MFCCS) {
        // speechpy.feature.filterbanks as speechpy.feature.mfe calls it (precise/vectorization.py:40-42; the package itself is not in
        // the reference tree: PARITY UNPINNED, its published algorithm is restated): mel points between 0 and sample_rate / 2, corner bins
        // floor((coefficients + 1) * hz / sample_rate) with coefficients = n_fft / 2 + 1, triangles without de-duplication.
        const double top2 = 1127.0 * log(1.0 + 0.5 * (double)c.sample_rate / 700.0);
        for (int i = 0; i < nf + 2; ++i) {
            const double m = (i == nf + 1) ? top2 : (double)i * (top2 / (double)(nf + 1));
            const double hz = 700.0 * (exp(m / 1127.0) - 1.0);
            grid[i] = (int)floor((double)(nb + 1) * hz / (double)c.sample_rate);
        }
    } else
    for (int i = 0; i < nf + 2; ++i) {
        // np.linspace(0, top, nf + 2): i * step, last element forced to stop
        double m = (i == nf + 1) ? top : (double)i * (top / (double)(nf + 1));
        double hz = 700.0 * (exp(m / 1127.0) - 1.0);
        long long raw = (long long)(hz * (double)nb / (double)c.sample_rate);
        if (i == 0) prev = raw - 1;
        shift = std::max(0LL, shift + prev + 1 - raw);
        grid[i] = (int)(raw + shift);
        prev = raw;
    }
    if (grid[nf + 1] > nb)
        return fail(PB_ERR_INVALID, "mel grid exceeds the spectrum (%d > %d bins): the reference's sonopy.filterbanks raises here", grid[nf + 1], nb);
    fb.assign((size_t)nf * nb, 0.0);
    mel.wrise.assign(nb, 0.f);
    mel.wfall.assign(nb, 0.f);
    for (int i = 0; i < nf; ++i) {
        int lo = grid[i], mid = grid[i + 1], hi = grid[i + 2];
        for (int k = lo; k < mid; ++k) fb[(size_t)i * nb + k] = (double)(k - lo) * (1.0 / (double)(mid - lo));
        for (int k = mid; k < hi; ++k) fb[(size_t)i * nb + k] = (double)(k - mid) * (-1.0 / (double)(hi - mid)) + 1.0;
        for (int k = lo; k < mid; ++k) mel.wrise[k] = (float)fb[(size_t)i * nb + k];
        for (int k = mid; k < hi; ++k) mel.wfall[k] = (float)fb[(size_t)i * nb + k];
    }
    return PB_OK;
}

static void build_cdf(Network& net) {
    // precise/threshold_decoder.py:38-43, :68-70 and functions.pdf (:104-108)
    const pb_config& c = net.cfg;
    const int resolution = 200;
    double lo = 0, hi = 0;
    for (int i = 0; i < c.n_thresholds; ++i) {
        double a = c.threshold_mu[i] + -4 * c.threshold_std[i], b = c.threshold_mu[i] + 4 * c.threshold_std[i];
        if (i == 0 || a < lo) lo = a;
        if (i == 0 || b > hi) hi = b;
    }
    net.min_out = (int)lo;
    net.max_out = (int)hi;
    const int range = net.max_out - net.min_out;
    const int num = resolution * range;
    net.cd.assign(std::max(num, 0), 0.0);
    if (num <= 0) return;
    const double step = num > 1 ? (double)(net.max_out - net.min_out) / (double)(num - 1) : 0.0;
    double run = 0.0;
    for (int j = 0; j < num; ++j) {
        double x = (j == num - 1 && num > 1) ? (double)net.max_out : (double)j * step + (double)net.min_out;
        double s = 0.0;
        for (int i = 0; i < c.n_thresholds; ++i) {
            double mu = c.threshold_mu[i], sd = c.threshold_std[i];
            double p = sd == 0 ? 0.0 : (1.0 / (sd * sqrt(2 * M_PI))) * exp(-((x - mu) * (x - mu)) / (2 * (sd * sd)));
            s = (i == 0) ? p : s + p;
        }
        run += s / (double)(resolution * c.n_thresholds);
        net.cd[j] = run;
    }
}

// The network fields of a configuration (pb_create checks hidden earlier, with the other sizes).
static int check_network(const pb_config& c) {
    if (c.hidden < 1) return fail(PB_ERR_INVALID, "hidden must be positive");
    if (c.n_thresholds < 1 || c.n_thresholds > PB_MAX_THRESHOLDS) return fail(PB_ERR_INVALID, "n_thresholds must be in [1, %d]", PB_MAX_THRESHOLDS);
    if (c.activation < 0 || c.activation > 1 || c.recurrent_activation < 0 || c.recurrent_activation > 1)
        return fail(PB_ERR_UNSUPPORTED, "unsupported GRU activation");
    return PB_OK;
}

// A network's decoder table (net.cd as built or replaced) and zeroed trigger array on the current device.
static cudaError_t upload_network_state(Network& net, size_t max_streams) {
    cudaError_t e = net.d_cd.upload(net.cd);
    if (e == cudaSuccess) e = net.trig.alloc(max_streams);
    if (e == cudaSuccess) e = cudaMemset(net.trig.get(), 0, max_streams * sizeof(int));
    return e;
}

static bool is_pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }

// cudaFuncAttributeMaxDynamicSharedMemorySize belongs to the kernel, not to a handle: handles with different geometries
// (n_filt, hidden, ...) coexist in one process, so only ever raise it -- to the largest size any handle has asked for.
template <typename K>
static cudaError_t ensure_dyn_smem(K kernel, size_t bytes) {
    static std::mutex mu;
    static std::map<std::pair<int, const void*>, size_t> granted;     // per (device, kernel): the attribute lives in the context
    int dev = 0;
    cudaError_t e0 = cudaGetDevice(&dev);
    if (e0 != cudaSuccess) return e0;
    std::lock_guard<std::mutex> lock(mu);
    size_t& cur = granted[std::make_pair(dev, (const void*)kernel)];
    if (bytes <= cur) return cudaSuccess;
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e == cudaSuccess) cur = bytes;
    return e;
}

// ------------------------------------------------------------------------------------------------
#define PB_API extern "C" __attribute__((visibility("default")))

PB_API int pb_abi_version(void) { return PB_ABI_VERSION; }
PB_API const char* pb_last_error(void) { return g_err; }
PB_API const char* pb_build_info(void) { return "precise_b200 sm_90a " __DATE__ " " __TIME__; }

PB_API int pb_config_default(pb_config* cfg) {
    if (!cfg) return fail(PB_ERR_INVALID, "cfg is null");
    memset(cfg, 0, sizeof(*cfg));
    cfg->abi_version = PB_ABI_VERSION;
    cfg->device = 0;
    cfg->max_streams = 1;
    cfg->chunk_samples = 1024;
    cfg->sample_rate = 16000;
    cfg->window_samples = 1600;
    cfg->hop_samples = 800;
    cfg->n_fft = 512;
    cfg->n_filt = 20;
    cfg->n_mfcc = 13;
    cfg->n_features = 29;
    cfg->use_delta = 0;
    cfg->vectorizer = PB_VEC_MFCCS;
    cfg->hidden = 20;
    cfg->activation = PB_ACT_LINEAR;
    cfg->recurrent_activation = PB_RACT_HARD_SIGMOID;
    cfg->n_thresholds = 1;
    cfg->threshold_mu[0] = 6.0;
    cfg->threshold_std[0] = 4.0;
    cfg->threshold_center = 0.2;
    cfg->sensitivity = 0.5;
    cfg->trigger_level = 3;
    return PB_OK;
}

PB_API void pb_destroy(pb_handle* h) {
    if (!h) return;
    cudaSetDevice(h->cfg.device);
    delete h;
}

PB_API int pb_create(const pb_config* cfg, pb_handle** out) {
    if (!cfg || !out) return fail(PB_ERR_INVALID, "null argument");
    *out = nullptr;
    const pb_config& c = *cfg;
    if (c.abi_version != PB_ABI_VERSION) return fail(PB_ERR_INVALID, "abi_version %d != %d", c.abi_version, PB_ABI_VERSION);
    if (c.max_streams < 1) return fail(PB_ERR_INVALID, "max_streams must be >= 1");
    if (c.chunk_samples < 1) return fail(PB_ERR_INVALID, "chunk_samples must be >= 1");
    if (c.sample_rate < 1 || c.window_samples < 1 || c.hop_samples < 1 || c.n_features < 1 || c.hidden < 1)
        return fail(PB_ERR_INVALID, "sample_rate, window_samples, hop_samples, n_features, hidden must be positive");
    if (c.vectorizer != PB_VEC_MFCCS && c.vectorizer != PB_VEC_MELS && c.vectorizer != PB_VEC_SPEECHPY_MFCCS) return fail(PB_ERR_INVALID, "unknown vectorizer %d", c.vectorizer);
    if (!is_pow2(c.n_fft) || c.n_fft < 64 || c.n_fft > 1024)
        return fail(PB_ERR_UNSUPPORTED, "n_fft %d: powers of two in [64, 1024] are implemented (512 is the reference default)", c.n_fft);
    if (c.n_filt < 1 || c.n_filt > 64 || c.n_mfcc < 1 || c.n_mfcc > 64) return fail(PB_ERR_UNSUPPORTED, "n_filt and n_mfcc must be in [1, 64]");
    int rc = check_network(c);
    if (rc != PB_OK) return rc;
    int ndev = 0;
    CK(cudaGetDeviceCount(&ndev));
    if (c.device < 0 || c.device >= ndev) return fail(PB_ERR_CUDA, "device %d not available (%d visible)", c.device, ndev);
    CK(cudaSetDevice(c.device));

    std::unique_ptr<pb_handle> h(new (std::nothrow) pb_handle());      // deleted, with this device current, on every early return
    if (!h) return fail(PB_ERR_CUDA, "out of host memory");
    h->cfg = c;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, c.device) == cudaSuccess) h->sm_count = prop.multiProcessorCount;
    h->used = std::min(c.n_fft, c.window_samples);
    h->n_bins = c.n_fft / 2 + 1;
    h->n_out = c.vectorizer == PB_VEC_MELS ? c.n_filt : std::min(c.n_filt, c.n_mfcc);
    h->feat = h->n_out * (c.use_delta ? 2 : 1);
    h->row_stride = (h->n_out + 3) & ~3;
    // speechpy's stack_frames yields floor((len - window) / hop) frames, one fewer than sonopy's framing: frame k is released one hop later
    h->rel_window = c.window_samples + (c.vectorizer == PB_VEC_SPEECHPY_MFCCS ? c.hop_samples : 0);
    h->ring_rows = c.n_features + (h->rel_window - h->used) / c.hop_samples + 2;
    h->tail_cap = (h->used + 7) & ~7;            // rows stay 16-byte aligned
    h->max_new = c.chunk_samples / c.hop_samples + 2;

    const size_t k1_big = c.n_fft > 512 ? k1_big_smem + 16 : 0;      // n_fft = 1024: power rows and FFT scratch in the dynamic tail
    h->k1_batch_smem = sizeof(K1Smem) + (size_t)h->n_out * c.n_filt * sizeof(float) + k1_big;
    h->k1_stream_smem = sizeof(K1StreamSmem) + (size_t)h->n_out * c.n_filt * sizeof(float) + k1_big;
    MelHost mel;
    rc = build_mel(c, h->n_bins, mel);
    if (rc != PB_OK) return rc;
    const std::vector<int>& grid = mel.grid;
    // piece schedule of the 16-lane mel stage (mfcc_fast.cuh): <= 8 bins each, never across a grid point
    std::vector<int> pieces, seg_first(c.n_filt + 2, 0);
    {
        auto add_range = [&](int lo, int hi) {
            for (int k = lo; k < hi; k += K1F_PIECE_LEN) pieces.push_back(k | (std::min(K1F_PIECE_LEN, hi - k) << 16));
        };
        for (int i = 0; i <= c.n_filt; ++i) {
            seg_first[i] = (int)pieces.size();
            add_range(grid[i], std::min(grid[i + 1], h->n_bins));
        }
        seg_first[c.n_filt + 1] = (int)pieces.size();
        add_range(0, std::min(grid[0], h->n_bins));                       // bins outside the grid: total power only
        add_range(grid[c.n_filt + 1], h->n_bins);
    }
    const int n_pieces = (int)pieces.size();
    h->npl = (n_pieces + 15) / 16;
    h->nol = (h->n_out + 15) / 16;
    h->maxc = 1;
    for (int j = 0; j < c.n_filt; ++j) h->maxc = std::max(h->maxc, seg_first[j + 2] - seg_first[j]);
    // ptab[q][e][lane]: piece p = lane + 16 q, entry e -> (byte offset of the bin in P, w_rise, w_fall, 0); padding -> zero bin
    std::vector<float4> ptab((size_t)h->npl * 128);
    for (int q = 0; q < h->npl; ++q)
        for (int e = 0; e < 8; ++e)
            for (int lane = 0; lane < 16; ++lane) {
                const int pidx = lane + 16 * q;
                int bin = K1F_ZERO_BIN;
                float wr = 0.f, wf = 0.f;
                if (pidx < n_pieces) {
                    const int start = pieces[pidx] & 0xffff, len = pieces[pidx] >> 16;
                    if (e < len) { bin = start + e; wr = mel.wrise[bin]; wf = mel.wfall[bin]; }
                }
                const int off = bin * 4;
                float offf; memcpy(&offf, &off, 4);
                ptab[((size_t)q * 8 + e) * 16 + lane] = make_float4(offf, wr, wf, 0.f);
            }
    // ctab[j][c]: partial slots summed into filter j: rise partials of segment j, fall partials (index + 64) of segment j + 1
    std::vector<unsigned char> ctab((size_t)c.n_filt * h->maxc, 128);
    for (int j = 0; j < c.n_filt; ++j) {
        int w = 0;
        for (int pp = seg_first[j]; pp < seg_first[j + 1]; ++pp) ctab[(size_t)j * h->maxc + w++] = (unsigned char)pp;
        for (int pp = seg_first[j + 1]; pp < seg_first[j + 2]; ++pp) ctab[(size_t)j * h->maxc + w++] = (unsigned char)(64 + pp);
    }
    h->fast_ok = c.n_fft == 512 && h->used == 512 && c.hop_samples % 8 == 0 && n_pieces <= 64 && h->npl <= 4;
    h->mma_ok = h->fast_ok && c.vectorizer == PB_VEC_MFCCS && c.n_filt <= MM_MAX_FILT && h->n_out <= MM_MAX_FILT && !c.use_delta &&
                c.chunk_samples % 8 == 0 && c.hop_samples >= 512 && c.chunk_samples >= c.hop_samples && c.chunk_samples <= 32760;
    const size_t k1_fast_tables = (size_t)h->npl * 128 * sizeof(float4) + (size_t)c.n_filt * 16 * h->nol * sizeof(float) +
                                  (((size_t)c.n_filt * h->maxc + 15) & ~(size_t)15);
    h->k1_fast_smem = K1F_WARPS * sizeof(K1FWarp) + k1_fast_tables;
    h->k1_pipe_smem = K1F_WARPS * sizeof(K1PWarp) + 256 * sizeof(float2) + k1_fast_tables;
    h->k1_ragged_smem = K1F_WARPS * sizeof(K1RWarp) + k1_fast_tables;
    // DCT-II, norm='ortho' (scipy.fftpack.dct as sonopy.mfcc_spec calls it), first n_out rows
    std::vector<float> dct((size_t)h->n_out * c.n_filt);
    for (int k = 0; k < h->n_out; ++k)
        for (int n = 0; n < c.n_filt; ++n) {
            double v = cos(M_PI * k * (2 * n + 1) / (2.0 * c.n_filt)) * sqrt(2.0 / c.n_filt);
            if (k == 0) v *= sqrt(0.5);
            dct[(size_t)k * c.n_filt + n] = (float)v;
        }
    std::vector<float2> tws(256), twp(16);
    for (int n2 = 0; n2 < 16; ++n2)
        for (int k1 = 0; k1 < 16; ++k1) {
            double a = 2.0 * M_PI * (double)(n2 * k1) / 256.0;
            tws[n2 * 16 + k1] = make_float2((float)cos(a), (float)-sin(a));
        }
    for (int k1 = 0; k1 < 16; ++k1) {
        double a = 2.0 * M_PI * (double)k1 / 512.0;
        twp[k1] = make_float2((float)cos(a), (float)sin(a));
    }
    std::vector<float2> twa(c.n_fft / 2);
    for (int k = 0; k < c.n_fft / 2; ++k) {
        double a = 2.0 * M_PI * (double)k / (double)c.n_fft;
        twa[k] = make_float2((float)cos(a), (float)-sin(a));
    }
    CK(h->d_wrise.upload(mel.wrise));
    CK(h->d_wfall.upload(mel.wfall));
    CK(h->d_grid.upload(grid));
    h->fb = std::move(mel.fb);
    CK(h->d_dct.upload(dct));
    CK(h->d_tw_stage.upload(tws));
    CK(h->d_tw_post.upload(twp));
    CK(h->d_tw_any.upload(twa));
    {
        std::vector<float> dct_t((size_t)c.n_filt * 16 * h->nol, 0.f);
        for (int k = 0; k < h->n_out; ++k)
            for (int n = 0; n < c.n_filt; ++n) dct_t[(size_t)n * 16 * h->nol + k] = dct[(size_t)k * c.n_filt + n];
        CK(h->d_dct_t.upload(dct_t));
    }
    CK(h->d_ptab.upload(ptab));
    CK(h->d_ctab.upload(ctab));
    const size_t S = (size_t)c.max_streams;
    CK(h->d_n_samples.alloc(S));
    CK(h->d_tail.alloc(S * h->tail_cap));
    CK(h->d_ring.alloc(S * h->ring_rows * h->row_stride));
    CK(cudaMemset(h->d_n_samples.get(), 0, S * sizeof(long long)));
    CK(cudaMemset(h->d_tail.get(), 0, S * h->tail_cap * sizeof(int16_t)));
    CK(cudaMemset(h->d_ring.get(), 0, S * h->ring_rows * h->row_stride * sizeof(float)));
    CK(h->d_count.alloc(1));
    CK(cudaMemset(h->d_count.get(), 0, sizeof(unsigned long long)));
    CK(ensure_dyn_smem(mfcc_batch_kernel<int16_t, true>, (size_t)(h->k1_batch_smem)));
    CK(ensure_dyn_smem(mfcc_batch_kernel<int16_t, false>, (size_t)(h->k1_batch_smem)));
    CK(ensure_dyn_smem(mfcc_batch_kernel<float, true>, (size_t)(h->k1_batch_smem)));
    CK(ensure_dyn_smem(mfcc_batch_kernel<float, false>, (size_t)(h->k1_batch_smem)));
    CK(ensure_dyn_smem(mfcc_fast_batch_kernel, (size_t)(h->k1_fast_smem)));
    CK(ensure_dyn_smem(mfcc_fast_stream_kernel<false>, (size_t)(h->k1_fast_smem)));
    CK(ensure_dyn_smem(mfcc_fast_stream_kernel<true>, (size_t)(h->k1_fast_smem)));
    CK(ensure_dyn_smem(mfcc_pipe_stream_kernel, (size_t)(h->k1_pipe_smem)));
    // K1P_CTAS_PER_SM CTAs of k1_pipe_smem each need the largest shared-memory carveout
    CK(cudaFuncSetAttribute(mfcc_pipe_stream_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
    CK(ensure_dyn_smem(mfcc_stream_kernel<true>, (size_t)(h->k1_stream_smem)));
    CK(ensure_dyn_smem(mfcc_stream_kernel<false>, (size_t)(h->k1_stream_smem)));
    CK(ensure_dyn_smem(mfcc_stream_kernel<false, true>, (size_t)(h->k1_stream_smem)));
    CK(ensure_dyn_smem(mfcc_ragged_stream_kernel, (size_t)(h->k1_ragged_smem)));
    CK(ensure_dyn_smem(mfcc_fast_corpus_kernel, (size_t)(h->k1_fast_smem)));
    CK(ensure_dyn_smem(mfcc_corpus_kernel, (size_t)(h->k1_batch_smem)));

    Network net;                     // slot 0: weights come with pb_load_weights
    net.cfg = c;
    build_cdf(net);
    CK(upload_network_state(net, S));
    h->models.push_back(std::move(net));
    *out = h.release();
    return PB_OK;
}

PB_API int64_t pb_mfcc_frames(const pb_handle* h, int64_t n) {
    if (!h) return 0;
    return n < h->rel_window ? 0 : (n - h->rel_window) / h->cfg.hop_samples + 1;
}
PB_API int32_t pb_feature_size(const pb_handle* h) { return h ? h->feat : 0; }
PB_API int32_t pb_mfcc_width(const pb_handle* h) { return h ? h->n_out : 0; }

PB_API int pb_get_filterbank(const pb_handle* h, double* out) {
    if (!h || !out) return fail(PB_ERR_INVALID, "null argument");
    memcpy(out, h->fb.data(), h->fb.size() * sizeof(double));
    return PB_OK;
}

PB_API int64_t pb_get_cdf(const pb_handle* h, double* out, int64_t capacity, int32_t* min_out, int32_t* max_out) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    const Network& net = h->models[0];
    if (min_out) *min_out = net.min_out;
    if (max_out) *max_out = net.max_out;
    if (out) memcpy(out, net.cd.data(), std::min<int64_t>(capacity, (int64_t)net.cd.size()) * sizeof(double));
    return (int64_t)net.cd.size();
}

PB_API int pb_set_cdf(pb_handle* h, const double* cd, int64_t len) {
    if (!h || !cd) return fail(PB_ERR_INVALID, "null argument");
    Network& net = h->models[0];
    if (len != (int64_t)net.cd.size()) return fail(PB_ERR_INVALID, "cdf length %lld != %zu", (long long)len, net.cd.size());
    CK(cudaSetDevice(h->cfg.device));
    memcpy(net.cd.data(), cd, len * sizeof(double));
    if (len) CK(cudaMemcpy(net.d_cd.get(), cd, len * sizeof(double), cudaMemcpyHostToDevice));
    return PB_OK;
}

// Networks gru_bank_kernel scores: H <= 24, feature_size F <= 16, no deltas.
static bool bank_fused(const Network& net, int F) {
    return net.cfg.hidden <= BANK_MAX_H && F <= BANK_MAX_F && !net.cfg.use_delta;
}

// fp16 hi / lo weight fragments of the fused family (gru_bank_kernel).  Column (nt, g) -> gate nt / 3,
// unit 8 (nt % 3) + g.  Recurrent weights: k-tile 0 = hidden units 0..15 as an m16n8k16 B fragment (b0: k = 2t, 2t + 1;
// b1: k = 2t + 8, 2t + 9), k-tile 1 = units 16..23 as an m16n8k8 one (b0 only).  Input weights: features 0..15 as one k16
// fragment.  Bias and dense weights padded to 24 units per gate.  Built on the host, then uploaded per bank model
// (upload_frag16) or copied into a pool slot (pb_pool_load).
struct Frag16 {
    std::vector<uint4> bf16, xf16;   // [2][MMA_NT][32], [MMA_NT][32]
    std::vector<float> mb, mw;       // [3][24], [24]
};

static void build_frag16(Frag16& fr, int H, int F, const float* kernel, const float* recurrent, const float* bias, const float* dense_w) {
    const int H3 = 3 * H;
    auto h2 = [](float lo16, float hi16) {
        const __half a = __float2half_rn(lo16), b = __float2half_rn(hi16);
        uint16_t ua, ub; memcpy(&ua, &a, 2); memcpy(&ub, &b, 2);
        return (uint32_t)ua | ((uint32_t)ub << 16);
    };
    auto res = [](float v) { return v - __half2float(__float2half_rn(v)); };
    std::vector<uint4>& bf16 = fr.bf16;
    bf16.assign((size_t)2 * MMA_NT * 32, uint4{});
    for (int kt = 0; kt < 2; ++kt)
        for (int nt = 0; nt < MMA_NT; ++nt)
            for (int lane = 0; lane < 32; ++lane) {
                const int g = lane >> 2, t = lane & 3, gate = nt / 3, unit = 8 * (nt % 3) + g;
                float b[2][2];
                for (int r = 0; r < 2; ++r)
                    for (int j = 0; j < 2; ++j) {
                        const int hu = 16 * kt + 8 * r + 2 * t + j;
                        b[r][j] = (unit < H && hu < H && !(kt == 1 && r == 1)) ? recurrent[(size_t)hu * H3 + gate * H + unit] : 0.f;
                    }
                bf16[((size_t)kt * MMA_NT + nt) * 32 + lane] = make_uint4(h2(b[0][0], b[0][1]), h2(b[1][0], b[1][1]),
                                                                          h2(res(b[0][0]), res(b[0][1])), h2(res(b[1][0]), res(b[1][1])));
            }
    std::vector<uint4>& xf16 = fr.xf16;
    xf16.assign((size_t)MMA_NT * 32, uint4{});
    for (int nt = 0; nt < MMA_NT; ++nt)
        for (int lane = 0; lane < 32; ++lane) {
            const int g = lane >> 2, t = lane & 3, gate = nt / 3, unit = 8 * (nt % 3) + g;
            float b[2][2];
            for (int r = 0; r < 2; ++r)
                for (int j = 0; j < 2; ++j) {
                    const int f = 8 * r + 2 * t + j;
                    b[r][j] = (unit < H && f < F) ? kernel[(size_t)f * H3 + gate * H + unit] : 0.f;
                }
            xf16[(size_t)nt * 32 + lane] = make_uint4(h2(b[0][0], b[0][1]), h2(b[1][0], b[1][1]),
                                                      h2(res(b[0][0]), res(b[0][1])), h2(res(b[1][0]), res(b[1][1])));
        }
    fr.mb.assign(72, 0.f);
    fr.mw.assign(24, 0.f);
    for (int gate = 0; gate < 3; ++gate)
        for (int u = 0; u < H; ++u) fr.mb[gate * 24 + u] = bias[gate * H + u];
    for (int u = 0; u < H; ++u) fr.mw[u] = dense_w[u];
}

static int upload_frag16(NetWeights& w, const Frag16& fr) {
    CK(w.bfrag16.upload(fr.bf16));
    CK(w.xfrag16.upload(fr.xf16));
    CK(w.mma_bias.upload(fr.mb));
    CK(w.mma_wd.upload(fr.mw));
    return PB_OK;
}

// Fragment-ordered, TF32-split weights of gru_wide_kernel: k = 8 s + t (+ 4) is x feature k (k < FP) or hidden unit k - FP;
// phase-1 column n = 8 nt + g is z unit n (n < HP) or r unit n - HP, phase-2 column n is candidate unit n.
static int upload_wide(NetWeights& w, int H, int F, const float* kernel, const float* recurrent, const float* bias) {
    const int H3 = 3 * H;
    auto tf32 = [](float x) { uint32_t u; memcpy(&u, &x, 4); u = (u + 0x1000u) & 0xffffe000u; float r; memcpy(&r, &u, 4); return r; };
    const int FP = (F + 7) & ~7, HP = (H + 15) & ~15, KS = (FP + HP) / 8;
    w.wg_fp = FP; w.wg_hp = HP;
    auto wv = [&](int k, int gate, int unit) -> float {
        if (unit >= H) return 0.f;
        if (k < FP) return k < F ? kernel[(size_t)k * H3 + gate * H + unit] : 0.f;
        const int hu = k - FP;
        return hu < H ? recurrent[(size_t)hu * H3 + gate * H + unit] : 0.f;
    };
    auto frag = [&](int s, int lane, int gate, int unit) {
        const int t = lane & 3;
        const float v0 = wv(8 * s + t, gate, unit), v1 = wv(8 * s + t + 4, gate, unit);
        const float h0 = tf32(v0), h1 = tf32(v1), l0 = tf32(v0 - h0), l1 = tf32(v1 - h1);
        uint4 r; memcpy(&r.x, &h0, 4); memcpy(&r.y, &h1, 4); memcpy(&r.z, &l0, 4); memcpy(&r.w, &l1, 4);
        return r;
    };
    std::vector<uint4> b1((size_t)KS * (HP / 4) * 32), b2((size_t)KS * (HP / 8) * 32);
    for (int s = 0; s < KS; ++s)
        for (int lane = 0; lane < 32; ++lane) {
            for (int nt = 0; nt < HP / 4; ++nt) {
                const int c = 8 * nt + (lane >> 2);
                b1[((size_t)s * (HP / 4) + nt) * 32 + lane] = frag(s, lane, c < HP ? 0 : 1, c % HP);
            }
            for (int nt = 0; nt < HP / 8; ++nt) b2[((size_t)s * (HP / 8) + nt) * 32 + lane] = frag(s, lane, 2, 8 * nt + (lane >> 2));
        }
    std::vector<float> wb((size_t)3 * HP, 0.f);
    for (int g3 = 0; g3 < 3; ++g3)
        for (int u = 0; u < H; ++u) wb[(size_t)g3 * HP + u] = bias[g3 * H + u];
    CK(w.wg_b1.upload(b1));
    CK(w.wg_b2.upload(b2));
    CK(w.wg_bias.upload(wb));
    return PB_OK;
}

// [W; U] of gru_tiled_kernel, its bias and the dense weights.
static int upload_tiled(NetWeights& w, int H, int F, const float* kernel, const float* recurrent, const float* bias, const float* dense_w) {
    const int H3 = 3 * H;
    std::vector<float> wcat((size_t)(F + H) * H3);
    memcpy(wcat.data(), kernel, (size_t)F * H3 * sizeof(float));
    memcpy(wcat.data() + (size_t)F * H3, recurrent, (size_t)H * H3 * sizeof(float));
    CK(w.wcat.upload(wcat));
    CK(w.bias.upload(std::vector<float>(bias, bias + H3)));
    CK(w.wd.upload(std::vector<float>(dense_w, dense_w + H)));
    return PB_OK;
}

// Builds every layout of net's new weights (F = the front end's feature size) and raises the kernels' shared-memory limits;
// only when all of that succeeded do they replace net's weights.  On failure net keeps what it had, weights or none.
// The current device is the handle's: the replaced weights are freed on it.
static int load_weights(Network& net, int F, const float* kernel, const float* recurrent, const float* bias,
                        const float* dense_w, float dense_b) {
    const pb_config& c = net.cfg;
    const int H = c.hidden;
    const size_t tiled_smem = (size_t)(F + 3 * H) * K2_TILE_STREAMS * sizeof(float);
    if (tiled_smem > 200 * 1024) return fail(PB_ERR_UNSUPPORTED, "feature_size + 3*hidden = %d is too large for the tiled GRU kernel", F + 3 * H);
    std::unique_ptr<NetWeights> w(new (std::nothrow) NetWeights());
    if (!w) return fail(PB_ERR_CUDA, "out of host memory");
    w->bd = dense_b;
    w->small_path = H == 20 && F == 13 && !c.use_delta && c.activation == PB_ACT_LINEAR && c.recurrent_activation == PB_RACT_HARD_SIGMOID;
    if (w->small_path) {
        memcpy(w->w_small.W, kernel, sizeof(w->w_small.W));
        memcpy(w->w_small.U, recurrent, sizeof(w->w_small.U));
        memcpy(w->w_small.b, bias, sizeof(w->w_small.b));
        memcpy(w->w_small.wd, dense_w, sizeof(w->w_small.wd));
        w->w_small.bd = dense_b;
    }
    w->wide_ok = !w->small_path && H <= WG_MAX_H && F <= WG_MAX_F;
    int rc = upload_tiled(*w, H, F, kernel, recurrent, bias, dense_w);
    if (rc == PB_OK && w->wide_ok) rc = upload_wide(*w, H, F, kernel, recurrent, bias);
    if (rc == PB_OK && bank_fused(net, F)) {
        Frag16 fr;
        build_frag16(fr, H, F, kernel, recurrent, bias, dense_w);
        rc = upload_frag16(*w, fr);
    }
    if (rc != PB_OK) return rc;
    if (w->wide_ok) {
        CK(ensure_dyn_smem(gru_wide_kernel<true>, wg_smem(w->wg_fp, w->wg_hp)));
        CK(ensure_dyn_smem(gru_wide_kernel<false>, wg_smem(w->wg_fp, w->wg_hp)));
    }
    if (!w->small_path) {
        CK(ensure_dyn_smem(gru_tiled_kernel<true>, tiled_smem));
        CK(ensure_dyn_smem(gru_tiled_kernel<false>, tiled_smem));
    }
    net.w = std::move(w);
    return PB_OK;
}

PB_API int pb_load_weights(pb_handle* h, const float* kernel, const float* recurrent, const float* bias,
                    const float* dense_w, float dense_b) {
    if (!h || !kernel || !recurrent || !bias || !dense_w) return fail(PB_ERR_INVALID, "null argument");
    CK(cudaSetDevice(h->cfg.device));
    return load_weights(h->models[0], h->feat, kernel, recurrent, bias, dense_w, dense_b);
}

// ------------------------------------------------------------------------------------------------
// profiling helpers
struct ProfScope {
    pb_handle* h; int slot; cudaStream_t s; int idx = -1;
    ProfScope(pb_handle* h_, int slot_, cudaStream_t s_) : h(h_), slot(slot_), s(s_) {
        if (!h->profiling) return;
        ProfSlot& p = h->prof[slot];
        if (p.used + 2 > (int)p.ev.size()) {
            if ((int)p.ev.size() >= 2 * PROFILE_POOL) {          // pool full: fold what we have
                for (int i = 0; i + 1 < p.used; i += 2) {
                    cudaEventSynchronize(p.ev[i + 1]);
                    float ms = 0; cudaEventElapsedTime(&ms, p.ev[i], p.ev[i + 1]); p.ms += ms;
                }
                p.used = 0;
            } else {
                cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b); p.ev.push_back(a); p.ev.push_back(b);
            }
        }
        idx = p.used; p.used += 2; p.launches++;
        cudaEventRecord(p.ev[idx], s);
    }
    ~ProfScope() { if (idx >= 0) cudaEventRecord(h->prof[slot].ev[idx + 1], s); }
};

PB_API int pb_debug_gru_mode(pb_handle* h, int mode) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    if (mode < 0 || mode > 2) return fail(PB_ERR_INVALID, "gru mode must be 0 (automatic), 1 (CUDA-core kernel) or 2 (tensor-core kernel)");
    h->models[0].gru_mode = mode;
    return PB_OK;
}

PB_API int pb_debug_k1_mode(pb_handle* h, int mode) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    if (mode < 0 || mode > 6 || mode == 1) return fail(PB_ERR_INVALID, "k1 mode must be 0 (automatic), 2 (FFT kernel, lean set-up, not pipelined), 3 (FFT kernel, 64-bit set-up), 4 (tensor-core DFT stage 2), 5 (both DFT stages on the tensor cores) or 6 (5 with a shuffle epilogue)");
    if (mode != 0 && h->ragged) return fail(PB_ERR_STATE, "k1 modes 2-6 need 16-byte-aligned stream state, which a handle loses with its first pb_update_ragged");
    if (mode >= 4 && !h->mma_ok) return fail(PB_ERR_UNSUPPORTED, "the tensor-core MFCC tick needs n_fft = 512 = frame length, hop >= 512 (a multiple of 8), chunk >= hop (a multiple of 8), n_filt <= 32, MFCC vectorizer");
    if ((mode == 2 || mode == 3) && !h->fast_ok) return fail(PB_ERR_UNSUPPORTED, "k1 modes 2 and 3 need the aligned geometry of the fast MFCC kernels");
    h->k1_mode = mode;
    return PB_OK;
}

// CPU model of the matrix-product DFT for one 512-sample frame (mfcc_tc.cuh: butterfly, operand tables and layout arithmetic
// of a tensor-core formulation).  No device needed; used by the CPU tests to pin that design.
PB_API int pb_debug_tc_dft_power(const int16_t* x512, double* power257) {
    if (!x512 || !power257) return fail(PB_ERR_INVALID, "null argument");
    tcd_host_power(x512, power257);
    return PB_OK;
}

// tables of the CPU model of the matrix-product MFCC, from the mel tables of configuration c (n_out MFCCs)
static void tcd_host_tables(const pb_config& c, int n_out, const MelHost& mel, std::vector<float4>& etab, std::vector<float>& dct,
                            float* tot_scale) {
    const float inv = 1.0f / 32768.0f, scale = inv * inv / (float)c.n_fft, pscale = scale / (TCD_A_SCALE * TCD_A_SCALE);
    tcd_build_etab(etab, mel.wrise, mel.wfall, mel.grid, c.n_filt, pscale);
    dct.assign((size_t)TCD_MAX_OUT * 24, 0.f);
    for (int k = 0; k < n_out; ++k)
        for (int j = 0; j < c.n_filt; ++j) {
            double v = cos(M_PI * k * (2 * j + 1) / (2.0 * c.n_filt)) * sqrt(2.0 / c.n_filt);
            if (k == 0) v *= sqrt(0.5);
            dct[(size_t)k * 24 + j] = (float)v;
        }
    *tot_scale = pscale;
}

// CPU model of the whole matrix-product MFCC for one frame: accumulator row (as above) + the epilogue (mel, log, DCT, c0) with
// the tables a handle of this configuration builds.  Needs no device.
PB_API int pb_debug_tc_mfcc_frame(const pb_config* cfg, const int16_t* x512, float* out) {
    if (!cfg || !x512 || !out) return fail(PB_ERR_INVALID, "null argument");
    if (cfg->n_fft != 512 || cfg->n_filt < 1 || cfg->n_filt > TCD_MAX_FILT || cfg->vectorizer != PB_VEC_MFCCS)
        return fail(PB_ERR_UNSUPPORTED, "the tensor-core MFCC model covers n_fft 512, n_filt <= %d, MFCC vectorizer", TCD_MAX_FILT);
    const int n_out = std::min(cfg->n_filt, cfg->n_mfcc);
    if (n_out > TCD_MAX_OUT) return fail(PB_ERR_UNSUPPORTED, "n_mfcc > %d", TCD_MAX_OUT);
    MelHost mel;
    const int rc = build_mel(*cfg, cfg->n_fft / 2 + 1, mel);
    if (rc != PB_OK) return rc;
    std::vector<float4> etab;
    std::vector<float> dct;
    float tot_scale = 0.f;
    tcd_host_tables(*cfg, n_out, mel, etab, dct, &tot_scale);
    float d[TCD_BLOCKS][64];
    tcd_host_accumulators(x512, d);
    tcd_host_epilogue(d, etab.data(), dct.data(), cfg->n_filt, n_out, tot_scale, out);
    return PB_OK;
}

// ... and of the formulation with both DFT stages as matrix products (mfcc_tc3.cuh): exact int16 split, stage-1 matrix passes, twiddle,
// fp16 split, stage-2 passes, its own epilogue order.  No device needed.  Test hook.
PB_API int pb_debug_tc3_mfcc_frame(const pb_config* cfg, const int16_t* x512, float* out, double* power257) {
    if (!cfg || !x512 || !out) return fail(PB_ERR_INVALID, "null argument");
    if (cfg->n_fft != 512 || cfg->n_filt < 1 || cfg->n_filt > TCD_MAX_FILT || cfg->vectorizer != PB_VEC_MFCCS)
        return fail(PB_ERR_UNSUPPORTED, "the tensor-core MFCC model covers n_fft 512, n_filt <= %d, MFCC vectorizer", TCD_MAX_FILT);
    const int n_out = std::min(cfg->n_filt, cfg->n_mfcc);
    if (n_out > TCD_MAX_OUT) return fail(PB_ERR_UNSUPPORTED, "n_mfcc > %d", TCD_MAX_OUT);
    MelHost mel;
    const int rc = build_mel(*cfg, cfg->n_fft / 2 + 1, mel);
    if (rc != PB_OK) return rc;
    std::vector<float4> etab;
    std::vector<float> dct;
    float tot_scale = 0.f;
    tcd_host_tables(*cfg, n_out, mel, etab, dct, &tot_scale);
    float d[TCD_BLOCKS][64];
    tc3_host_accumulators(x512, d);
    tc3_host_epilogue(d, mel.wrise, mel.wfall, mel.grid, dct.data(), cfg->n_filt, n_out, tot_scale, out);
    if (power257) {
        const double inv = 1.0 / ((double)TCD_A_SCALE * (double)TCD_A_SCALE);
        for (int b = 0; b < TCD_BLOCKS; ++b)
            for (int half = 0; half < 2; ++half)
                for (int m = 0; m < 16; ++m) {
                    const int k = tcd_col_bin(b, 32 * half + m);
                    if (k < 0) continue;
                    const double re = d[b][32 * half + m], im = d[b][32 * half + 16 + m];
                    power257[k] = (k == 0 || k == 256) ? re * re * inv : (re * re + im * im) * inv;
                }
    }
    return PB_OK;
}

// CPU model of the mma.sync MFCC tick's DFT (mfcc_mma.cuh: its fragment tables, splits and bin assembly) for one frame.  Test hook.
PB_API int pb_debug_mma_dft_power(const int16_t* x512, double* power257) {
    if (!x512 || !power257) return fail(PB_ERR_INVALID, "null argument");
    mm_host_power(x512, power257);
    return PB_OK;
}

PB_API int pb_debug_force_generic(pb_handle* h, int on) { if (!h) return fail(PB_ERR_INVALID, "null handle"); h->force_generic = on != 0; return PB_OK; }

PB_API int pb_profile_enable(pb_handle* h, int on) { if (!h) return fail(PB_ERR_INVALID, "null handle"); h->profiling = on != 0; return PB_OK; }

PB_API int pb_profile_reset(pb_handle* h) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    for (auto& p : h->prof) { p.used = 0; p.ms = 0; p.launches = 0; }
    return PB_OK;
}

PB_API int pb_profile_read(pb_handle* h, double ms[4], uint64_t launches[4]) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    CK(cudaSetDevice(h->cfg.device));
    for (int s = 0; s < N_PROFILE_SLOTS; ++s) {
        ProfSlot& p = h->prof[s];
        for (int i = 0; i + 1 < p.used; i += 2) {
            CK(cudaEventSynchronize(p.ev[i + 1]));
            float t = 0; CK(cudaEventElapsedTime(&t, p.ev[i], p.ev[i + 1])); p.ms += t;
        }
        p.used = 0;
        if (ms) ms[s] = p.ms;
        if (launches) launches[s] = p.launches;
    }
    return PB_OK;
}

// ------------------------------------------------------------------------------------------------
static MelTables mel_tables(const pb_handle* h) {
    MelTables t;
    t.w_rise = h->d_wrise.get(); t.w_fall = h->d_wfall.get(); t.grid = h->d_grid.get(); t.dct = h->d_dct.get();
    t.tw_stage = h->d_tw_stage.get(); t.tw_post = h->d_tw_post.get();
    t.n_bins = h->n_bins; t.n_filt = h->cfg.n_filt; t.n_out = h->n_out;
    t.mels_only = h->cfg.vectorizer == PB_VEC_MELS;
    t.n_fft = h->cfg.n_fft; t.tw_any = h->d_tw_any.get();
    return t;
}

static FastTables fast_tables(const pb_handle* h) {
    FastTables f;
    f.ptab = h->d_ptab.get(); f.ctab = h->d_ctab.get(); f.dct_t = h->d_dct_t.get();
    f.npl = h->npl; f.maxc = h->maxc; f.nol = h->nol;
    return f;
}

static StreamState stream_state(const pb_handle* h) {
    StreamState st;
    st.n_samples = h->d_n_samples.get(); st.tail = h->d_tail.get(); st.ring = h->d_ring.get();
    st.tail_cap = h->tail_cap; st.ring_rows = h->ring_rows; st.row_stride = h->row_stride;
    return st;
}

// TriggerDetector's refractory count -(8 * 2048) // chunk_size for chunk_size in bytes (>= 1), Python floor division.
static int trigger_reset(long long bytes) {
    long long q = -(8 * 2048) / bytes;                            // C truncates toward zero ...
    if ((-(8 * 2048)) % bytes != 0) q -= 1;                       // ... python floors
    return (int)q;
}

static DecodeParams decode_params(const Network& net) {
    const pb_config& c = net.cfg;
    DecodeParams d;
    d.cd = net.d_cd.get(); d.cd_len = (int)net.cd.size();
    d.min_out = net.min_out; d.out_range = net.max_out - net.min_out;
    d.center = c.threshold_center;
    d.hot_threshold = 1.0 - c.sensitivity;
    d.trigger_level = c.trigger_level;
    d.trigger_reset = trigger_reset(2LL * c.chunk_samples);        // TriggerDetector.chunk_size is in bytes
    d.legacy_f64 = c.decode_legacy_f64 != 0;
    return d;
}

// What a stream of net uses until pb_set_stream_trigger sets it: the model's own sensitivity and trigger_level, and the
// handle's chunk in bytes (capped at INT32_MAX, where the refractory count is -1 as for any chunk above 16 384 B).
static StreamTrig default_trig(const Network& net) {
    return StreamTrig{net.cfg.sensitivity, net.cfg.trigger_level, (int32_t)std::min<long long>(2LL * net.cfg.chunk_samples, INT32_MAX)};
}

static TrigRec trig_record(const StreamTrig& v) {
    return TrigRec{1.0 - v.sensitivity, v.trigger_level, trigger_reset(v.chunk_bytes)};
}

// A model with per-stream settings: its scan (K2Out o) writes raw and conf only, and trigger_kernel's slot nt, filled here from
// o, updates the trigger, fired and count afterwards.
static void defer_trigger(TrigTick& t, int& nt, const Network& net, unsigned route_bit, K2Out& o) {
    t.conf[nt] = o.conf; t.fired[nt] = o.fired; t.count[nt] = o.count; t.trig[nt] = o.trig;
    t.rec[nt] = net.trig_rec.get(); t.route_bit[nt] = route_bit;
    ++nt;
    o.trig = nullptr; o.fired = nullptr; o.count = nullptr;
}

// trigger_kernel over the nt deferred models of a tick; runs after their scans, on the same stream.
static int launch_trigger(const TrigTick& t, int nt, cudaStream_t s) {
    if (nt == 0 || t.n == 0) return PB_OK;
    trigger_kernel<<<dim3((unsigned)((t.n + 255) / 256), (unsigned)nt), 256, 0, s>>>(t);
    CK(cudaGetLastError());
    return PB_OK;
}

template <typename T>
static int mfcc_impl(pb_handle* h, const T* d_in, int64_t n_streams, int64_t L, float* d_out, cudaStream_t s, float scale) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    if (n_streams < 0 || L < 0) return fail(PB_ERR_INVALID, "negative size");
    if (L == 0 && n_streams > 0) return fail(PB_ERR_INVALID, "Cannot vectorize empty audio!");   // vectorization.py:48-49
    const int64_t nf = pb_mfcc_frames(h, L), total = nf * n_streams;
    if (total == 0) return PB_OK;
    if (!d_in || !d_out) return fail(PB_ERR_INVALID, "null buffer");
    CK(cudaSetDevice(h->cfg.device));
    const bool pairs = (L % 2 == 0) && (h->cfg.hop_samples % 2 == 0) && (h->used % 2 == 0) &&
                       ((uintptr_t)d_in % (2 * sizeof(T)) == 0);
    const int64_t tiles = (total + K1_TILE - 1) / K1_TILE;
    const int grid = (int)std::min<int64_t>(tiles, (int64_t)h->sm_count * 4);
    ProfScope ps(h, 0, s);
    if (sizeof(T) == 2 && h->fast_ok && L % 8 == 0 && (uintptr_t)d_in % 16 == 0 && !h->force_generic) {
        const int64_t pairs2 = (total + 1) / 2;
        const int gridf = (int)std::min<int64_t>((pairs2 + K1F_WARPS - 1) / K1F_WARPS, (int64_t)h->sm_count * 4);
        mfcc_fast_batch_kernel<<<gridf, K1F_THREADS, h->k1_fast_smem, s>>>((const int16_t*)d_in, L, nf, total, h->cfg.hop_samples, scale,
                                                                           mel_tables(h), fast_tables(h), d_out);
    } else if (pairs)
        mfcc_batch_kernel<T, true><<<grid, K1_THREADS, h->k1_batch_smem, s>>>(d_in, L, nf, total, h->cfg.hop_samples, h->used, scale, mel_tables(h), d_out);
    else
        mfcc_batch_kernel<T, false><<<grid, K1_THREADS, h->k1_batch_smem, s>>>(d_in, L, nf, total, h->cfg.hop_samples, h->used, scale, mel_tables(h), d_out);
    CK(cudaGetLastError());
    return PB_OK;
}

PB_API int pb_mfcc(pb_handle* h, const int16_t* d_pcm, int64_t n_streams, int64_t L, float* d_out, void* stream) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    const float inv = 1.0f / 32768.0f;
    return mfcc_impl<int16_t>(h, d_pcm, n_streams, L, d_out, (cudaStream_t)stream, inv * inv / (float)h->cfg.n_fft);
}

PB_API int pb_mfcc_f32(pb_handle* h, const float* d_audio, int64_t n_streams, int64_t L, float* d_out, void* stream) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    return mfcc_impl<float>(h, d_audio, n_streams, L, d_out, (cudaStream_t)stream, 1.0f / (float)h->cfg.n_fft);
}

// Model slot `slot` of a gru_bank_kernel launch: network net, scored with its decoder into o.
static void set_bank_slot(BankParams& P, int slot, const Network& net, const K2Out& o) {
    const NetWeights& nw = *net.w;
    BankModelW& w = P.w[slot];
    w.bfrag = nw.bfrag16.get(); w.xfrag = nw.xfrag16.get(); w.bias = nw.mma_bias.get(); w.wd = nw.mma_wd.get(); w.bd = nw.bd;
    w.act = net.cfg.activation; w.ract = net.cfg.recurrent_activation;
    P.dp[slot] = decode_params(net);
    P.o[slot] = o;
}

template <int NM, bool RING, bool KERAS_ACT>
static int launch_bank_act(const BankParams& P, const K2In& in, int64_t n, cudaStream_t s) {
    constexpr size_t smem = (size_t)NM * BANK_MODEL_SMEM + (bank_stages(NM, RING) ? BANK_STAGE_SMEM : 0);
    if constexpr (smem > 48 * 1024) CK(ensure_dyn_smem(gru_bank_kernel<NM, RING, KERAS_ACT>, smem));      // above the default limit
    const int per_cta = (MMA_THREADS / 32) * 16;
    gru_bank_kernel<NM, RING, KERAS_ACT><<<(int)((n + per_cta - 1) / per_cta), MMA_THREADS, smem, s>>>(P, in, n);
    CK(cudaGetLastError());
    return PB_OK;
}

// One model with Keras's GRU defaults (the networks Precise trains) runs with its activation pair compiled in.  Banks keep
// the run-time dispatch: with compiled-in activations ptxas interleaves the models' chains and needs up to 255 registers,
// spilling from NM = 4 on.
template <int NM, bool RING>
static int launch_bank_nm(const BankParams& P, const K2In& in, int64_t n, cudaStream_t s) {
    if constexpr (NM == 1)
        if (P.w[0].act == PB_ACT_LINEAR && P.w[0].ract == PB_RACT_HARD_SIGMOID) return launch_bank_act<1, RING, true>(P, in, n, s);
    return launch_bank_act<NM, RING, false>(P, in, n, s);
}

// Scores network net (which has weights; F = the front end's feature size) with its decoder into o.
static int launch_gru_kernels(const Network& net, int F, const K2In& in, bool ring, int64_t n, const K2Out& o, cudaStream_t s) {
    const NetWeights& nw = *net.w;
    const pb_config& c = net.cfg;
    const DecodeParams dp = decode_params(net);
    if (nw.small_path && n <= K2_WARP_PATH_MAX && net.gru_mode == 0) {                 // latency path: a warp per stream
        const int grid = (int)((n + 3) / 4);
        if (ring) gru_warp_kernel<20, 13, true><<<grid, 128, 0, s>>>(nw.w_small, in, n, dp, o);
        else gru_warp_kernel<20, 13, false><<<grid, 128, 0, s>>>(nw.w_small, in, n, dp, o);
    } else if (nw.small_path && net.gru_mode != 1) {              // tensor-core scan (mma.sync fp16 x 3): the bank kernel with one model
        BankParams P{};
        set_bank_slot(P, 0, net, o);
        return ring ? launch_bank_nm<1, true>(P, in, n, s) : launch_bank_nm<1, false>(P, in, n, s);
    } else if (nw.small_path) {
        const int per_cta = K2_SMALL_THREADS * K2_NS;
        const int grid = (int)((n + per_cta - 1) / per_cta);
        if (ring && o.route) gru_small_kernel<20, 13, true, true><<<grid, K2_SMALL_THREADS, 0, s>>>(nw.w_small, in, n, dp, o);
        else if (ring) gru_small_kernel<20, 13, true><<<grid, K2_SMALL_THREADS, 0, s>>>(nw.w_small, in, n, dp, o);
        else gru_small_kernel<20, 13, false><<<grid, K2_SMALL_THREADS, 0, s>>>(nw.w_small, in, n, dp, o);
    } else if (nw.wide_ok && net.gru_mode != 1) {                 // tensor-core scan (mma.sync 3xTF32) for other networks
        GruWideW w;
        w.b1 = nw.wg_b1.get(); w.b2 = nw.wg_b2.get(); w.bias = nw.wg_bias.get(); w.wd = nw.wd.get(); w.bd = nw.bd;
        w.H = c.hidden; w.F = F; w.FP = nw.wg_fp; w.HP = nw.wg_hp; w.act = c.activation; w.ract = c.recurrent_activation;
        const int grid = (int)((n + WG_STREAMS - 1) / WG_STREAMS);
        const size_t smem = wg_smem(w.FP, w.HP);
        if (ring) gru_wide_kernel<true><<<grid, WG_THREADS, smem, s>>>(w, in, n, dp, o);
        else gru_wide_kernel<false><<<grid, WG_THREADS, smem, s>>>(w, in, n, dp, o);
    } else {
        GruTiledW w;
        w.wcat = nw.wcat.get(); w.bias = nw.bias.get(); w.wd = nw.wd.get(); w.bd = nw.bd;
        w.H = c.hidden; w.F_in = F; w.act = c.activation; w.ract = c.recurrent_activation;
        const size_t smem = (size_t)(w.F_in + 3 * w.H) * K2_TILE_STREAMS * sizeof(float);
        const int grid = (int)((n + K2_TILE_STREAMS - 1) / K2_TILE_STREAMS);
        if (ring) gru_tiled_kernel<true><<<grid, K2_TILE_THREADS, smem, s>>>(w, in, n, dp, o);
        else gru_tiled_kernel<false><<<grid, K2_TILE_THREADS, smem, s>>>(w, in, n, dp, o);
    }
    CK(cudaGetLastError());
    return PB_OK;
}

static int launch_gru(pb_handle* h, const Network& net, const K2In& in, bool ring, int64_t n, const K2Out& o, cudaStream_t s) {
    ProfScope ps(h, 1, s);
    return launch_gru_kernels(net, h->feat, in, ring, n, o, s);
}

PB_API int pb_predict(pb_handle* h, const float* d_inputs, int64_t n, float* d_out, float* d_logit, void* stream) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    if (!h->models[0].w) return fail(PB_ERR_STATE, "pb_load_weights has not been called");
    if (n < 0) return fail(PB_ERR_INVALID, "negative n");
    if (n == 0) return PB_OK;
    if (!d_inputs || !d_out) return fail(PB_ERR_INVALID, "null buffer");
    CK(cudaSetDevice(h->cfg.device));
    K2In in{};
    in.inputs = d_inputs; in.row_stride = h->feat; in.T = h->cfg.n_features; in.F_base = h->n_out; in.use_delta = 0;
    K2Out o{};
    o.raw = d_out; o.logit = d_logit;
    return launch_gru(h, h->models[0], in, false, n, o, (cudaStream_t)stream);
}

PB_API int pb_decode(pb_handle* h, const float* d_raw, int64_t n, double* d_conf, void* stream) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    if (n < 0) return fail(PB_ERR_INVALID, "negative n");
    if (n == 0) return PB_OK;
    if (!d_raw || !d_conf) return fail(PB_ERR_INVALID, "null buffer");
    CK(cudaSetDevice(h->cfg.device));
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope ps(h, 2, s);
    decode_kernel<<<(int)((n + 255) / 256), 256, 0, s>>>(d_raw, n, decode_params(h->models[0]), d_conf);
    CK(cudaGetLastError());
    return PB_OK;
}

static int check_tick(pb_handle* h, const void* pcm, int64_t n) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    if (n < 0 || n > h->cfg.max_streams) return fail(PB_ERR_INVALID, "n = %lld outside [0, max_streams = %d]", (long long)n, h->cfg.max_streams);
    if (n > 0 && !pcm) return fail(PB_ERR_INVALID, "null pcm");
    return PB_OK;
}

static int ensure_mma_tables(pb_handle* h) {
    if (h->d_mm_b1.get()) return PB_OK;
    std::vector<uint2> b1, b2;
    std::vector<float2> tw;
    mm_build_tables(b1, b2, tw);
    CK(h->d_mm_b2.upload(b2));
    CK(h->d_mm_tw.upload(tw));
    CK(h->d_mm_recs.alloc((size_t)h->cfg.max_streams * (size_t)std::max(1, h->max_new)));
    CK(h->d_mm_counters.alloc(2));
    CK(cudaMemset(h->d_mm_counters.get(), 0, 2 * sizeof(unsigned int)));
    CK(ensure_dyn_smem(mfcc_mma_kernel<false, false>, sizeof(MmSmem)));
    CK(ensure_dyn_smem(mfcc_mma_kernel<true, false>, sizeof(MmSmem)));
    CK(ensure_dyn_smem(mfcc_mma_kernel<true, true>, sizeof(MmSmem)));
    CK(h->d_mm_b1.upload(b1));                           // last: its presence marks the set as complete
    return PB_OK;
}

// K1 of a ragged tick: item i's chunk is d_pcm[d_offsets[i] .. d_offsets[i + 1]) (d_offsets null: the uniform tick's
// d_pcm[i * chunk_samples ..), max_len = chunk_samples), lengths clamped to [0, max_len].  The tick runs as rounds of at most 6 hops
// per stream, so no stream completes more than 8 frames in one launch; to the state machine the rounds are separate ticks
// (Listener.update_vectors is chunking-independent).  Any alignment of offsets, lengths and sample counts.
static int launch_ragged_mfcc(pb_handle* h, const int16_t* d_pcm, const int64_t* d_offsets, int64_t max_len, const int32_t* d_ids,
                              int64_t n, cudaStream_t s) {
    const float inv = 1.0f / 32768.0f, scale = inv * inv / (float)h->cfg.n_fft;
    const StreamState st = stream_state(h);
    RaggedIn rg;
    rg.offsets = reinterpret_cast<const long long*>(d_offsets);
    rg.max_len = max_len;
    rg.chunk = h->cfg.chunk_samples;
    rg.sub = 6 * h->cfg.hop_samples;
    const bool fast = h->fast_ok && !h->force_generic;
    const int64_t warps_total = (int64_t)h->sm_count * 4 * K1F_WARPS;
    const int spw = (int)std::max<int64_t>(1, std::min<int64_t>(K1F_STREAMS_PER_WARP, (n + warps_total - 1) / warps_total));
    const int64_t tilesf = (n + spw - 1) / spw;
    const int gridf = (int)std::min<int64_t>((tilesf + K1F_WARPS - 1) / K1F_WARPS, (int64_t)h->sm_count * 4);
    const int grid = (int)std::min<int64_t>((n + K1_STREAMS_PER_CTA - 1) / K1_STREAMS_PER_CTA, (int64_t)h->sm_count * 4);
    ProfScope ps(h, 0, s);
    for (int64_t off = 0; off < max_len; off += rg.sub) {
        rg.round_off = off;
        if (fast)
            mfcc_ragged_stream_kernel<<<gridf, K1F_THREADS, h->k1_ragged_smem, s>>>(d_pcm, rg, d_ids, (int)n, h->cfg.hop_samples, spw, scale,
                                                                                   mel_tables(h), fast_tables(h), st);
        else
            mfcc_stream_kernel<false, true><<<grid, K1_THREADS, h->k1_stream_smem, s>>>(d_pcm, d_ids, (int)n, 0, 0, h->cfg.hop_samples, h->used,
                                                                                       scale, mel_tables(h), st, rg);
        CK(cudaGetLastError());
    }
    return PB_OK;
}

static int launch_stream_mfcc(pb_handle* h, const int16_t* d_pcm, const int32_t* d_ids, int64_t n, cudaStream_t s) {
    if (h->ragged) return launch_ragged_mfcc(h, d_pcm, nullptr, h->cfg.chunk_samples, d_ids, n, s);
    const bool pairs = (h->cfg.chunk_samples % 2 == 0) && (h->cfg.hop_samples % 2 == 0) && (h->used % 2 == 0) &&
                       ((uintptr_t)d_pcm % 4 == 0);
    const int64_t tiles = (n + K1_STREAMS_PER_CTA - 1) / K1_STREAMS_PER_CTA;
    const int grid = (int)std::min<int64_t>(tiles, (int64_t)h->sm_count * 4);
    const float inv = 1.0f / 32768.0f, scale = inv * inv / (float)h->cfg.n_fft;
    const StreamState st = stream_state(h);
    ProfScope ps(h, 0, s);
    if (h->k1_mode >= 4 && h->mma_ok && (uintptr_t)d_pcm % 16 == 0 && !h->force_generic) {
        int rc = ensure_mma_tables(h);
        if (rc != PB_OK) return rc;
        MmTables t;
        t.b1 = h->d_mm_b1.get(); t.b2 = h->d_mm_b2.get(); t.tw = h->d_mm_tw.get();
        t.pscale = inv * inv / (float)h->cfg.n_fft * 1024.f;             // the accumulators hold 2^-5 X
        const int par = h->mm_parity;
        h->mm_parity ^= 1;
        MmRec* recs = h->d_mm_recs.get();
        unsigned int* counters = h->d_mm_counters.get();
        mfcc_mma_plan_kernel<<<(int)((n + MM_PLAN_THREADS - 1) / MM_PLAN_THREADS), MM_PLAN_THREADS, 0, s>>>(
            d_pcm, d_ids, (int)n, h->cfg.chunk_samples, h->cfg.hop_samples, st, recs, counters, par);
        const int64_t max_tiles = (n * std::max(1, h->max_new) + MM_FRAMES - 1) / MM_FRAMES;
        const int gm = (int)std::min<int64_t>((max_tiles + MM_WARPS - 1) / MM_WARPS, h->sm_count);
        if (h->k1_mode == 4)
            mfcc_mma_kernel<false, false><<<gm, MM_THREADS, sizeof(MmSmem), s>>>(t, mel_tables(h), recs, counters, par);
        else if (h->k1_mode == 5)
            mfcc_mma_kernel<true, false><<<gm, MM_THREADS, sizeof(MmSmem), s>>>(t, mel_tables(h), recs, counters, par);
        else
            mfcc_mma_kernel<true, true><<<gm, MM_THREADS, sizeof(MmSmem), s>>>(t, mel_tables(h), recs, counters, par);
    } else if (h->fast_ok && h->max_new <= 8 && h->cfg.chunk_samples % 8 == 0 && (uintptr_t)d_pcm % 16 == 0 && !h->force_generic) {
        // streams per warp tile: 16 at scale; fewer when the batch cannot fill the machine's warps.  Every mode keeps this
        // tiling: a frame's half-warp, and with it the order of its mel16 sums, follows from its place in the tile
        const int64_t warps_total = (int64_t)h->sm_count * 4 * K1F_WARPS;
        const int spw = (int)std::max<int64_t>(1, std::min<int64_t>(K1F_STREAMS_PER_WARP, (n + warps_total - 1) / warps_total));
        const int64_t tilesf = (n + spw - 1) / spw;
        const int gridf = (int)std::min<int64_t>((tilesf + K1F_WARPS - 1) / K1F_WARPS, (int64_t)h->sm_count * 4);
        if (h->k1_mode == 0) {                   // default: the pipelined kernel (bit-identical rows, tails and counts to mode 2)
            const int gridp = (int)std::min<int64_t>((tilesf + K1F_WARPS - 1) / K1F_WARPS, (int64_t)h->sm_count * K1P_CTAS_PER_SM);
            mfcc_pipe_stream_kernel<<<gridp, K1F_THREADS, h->k1_pipe_smem, s>>>(d_pcm, d_ids, (int)n, h->cfg.chunk_samples, h->cfg.hop_samples, spw, scale,
                                                                              mel_tables(h), fast_tables(h), st);
        } else if (h->k1_mode != 3)              // the kernel mode 0 replaced: 32-bit per-pass set-up; 3 = its 64-bit original
            mfcc_fast_stream_kernel<true><<<gridf, K1F_THREADS, h->k1_fast_smem, s>>>(d_pcm, d_ids, (int)n, h->cfg.chunk_samples, h->cfg.hop_samples, spw, scale,
                                                                                      mel_tables(h), fast_tables(h), st);
        else
            mfcc_fast_stream_kernel<false><<<gridf, K1F_THREADS, h->k1_fast_smem, s>>>(d_pcm, d_ids, (int)n, h->cfg.chunk_samples, h->cfg.hop_samples, spw, scale,
                                                                                       mel_tables(h), fast_tables(h), st);
    } else if (h->max_new > 8) {
        // A chunk that completes more than 8 frames per stream: consecutive sub-chunks of at most 6 hops (<= 8 frames each) through the
        // generic kernel -- to the state machine they are separate ticks (Listener.update_vectors is chunking-independent); the network
        // runs once, after the last one.
        const int sub = std::max(1, 6 * h->cfg.hop_samples);
        for (int off = 0; off < h->cfg.chunk_samples; off += sub)
            mfcc_stream_kernel<false><<<grid, K1_THREADS, h->k1_stream_smem, s>>>(d_pcm + off, d_ids, (int)n, std::min(sub, h->cfg.chunk_samples - off),
                                                                                    h->cfg.chunk_samples, h->cfg.hop_samples, h->used, scale, mel_tables(h), st, RaggedIn{});
    } else if (pairs)
        mfcc_stream_kernel<true><<<grid, K1_THREADS, h->k1_stream_smem, s>>>(d_pcm, d_ids, (int)n, h->cfg.chunk_samples, h->cfg.chunk_samples, h->cfg.hop_samples, h->used, scale, mel_tables(h), st, RaggedIn{});
    else
        mfcc_stream_kernel<false><<<grid, K1_THREADS, h->k1_stream_smem, s>>>(d_pcm, d_ids, (int)n, h->cfg.chunk_samples, h->cfg.chunk_samples, h->cfg.hop_samples, h->used, scale, mel_tables(h), st, RaggedIn{});
    CK(cudaGetLastError());
    return PB_OK;
}

static HistPool hist_pool(const pb_handle* h) {
    HistPool P;
    P.rows = h->d_hist.get(); P.row_of = h->d_hist_row.get(); P.start = h->d_hist_start.get(); P.cap = h->hist_cap;
    return P;
}

// History half of a tick, before its K1 (the pre-tick n_samples): item i's chunk as K1 takes it (d_offsets null: the uniform
// tick's d_pcm[i * chunk_samples ..)) goes to the row of its stream.  Nothing without a pool.
static int append_history(pb_handle* h, const int16_t* d_pcm, const int64_t* d_offsets, int64_t max_len, const int32_t* d_ids,
                          int64_t n, cudaStream_t s) {
    if (!h->history) return PB_OK;
    RaggedIn rg{};
    rg.offsets = reinterpret_cast<const long long*>(d_offsets);
    rg.max_len = max_len;
    rg.chunk = h->cfg.chunk_samples;
    rg.sub = (int)std::min<int64_t>(max_len, INT32_MAX);
    const int per = HIST_THREADS / 32;
    ProfScope ps(h, 3, s);
    history_append_kernel<<<(unsigned)((n + per - 1) / per), HIST_THREADS, 0, s>>>(d_pcm, rg, d_ids, (int)n, h->d_n_samples.get(),
                                                                                  hist_pool(h));
    CK(cudaGetLastError());
    return PB_OK;
}

// A uniform tick's K1 with its history append first.
static int tick_mfcc(pb_handle* h, const int16_t* d_pcm, const int32_t* d_ids, int64_t n, cudaStream_t s) {
    const int rc = append_history(h, d_pcm, nullptr, h->cfg.chunk_samples, d_ids, n, s);
    return rc != PB_OK ? rc : launch_stream_mfcc(h, d_pcm, d_ids, n, s);
}

PB_API int pb_update_vectors(pb_handle* h, const int16_t* d_pcm, const int32_t* d_ids, int64_t n, void* stream) {
    int rc = check_tick(h, d_pcm, n);
    if (rc != PB_OK || n == 0) return rc;
    CK(cudaSetDevice(h->cfg.device));
    return tick_mfcc(h, d_pcm, d_ids, n, (cudaStream_t)stream);
}

// Where a stream tick's network kernels read the window of item i: stream d_ids[i] (i when d_ids is null) of the handle's ring.
static K2In stream_k2in(const pb_handle* h, const int32_t* d_ids) {
    K2In in{};
    in.ring = h->d_ring.get(); in.n_samples = h->d_n_samples.get(); in.ids = d_ids;
    in.ring_rows = h->ring_rows; in.row_stride = h->row_stride; in.window = h->rel_window; in.hop = h->cfg.hop_samples;
    in.T = h->cfg.n_features; in.F_base = h->n_out; in.use_delta = h->cfg.use_delta;
    return in;
}

// The network half of pb_update: slot 0 scores the windows of the n streams (its warp-per-stream kernel up to 8 192 streams).
static int score_model0(pb_handle* h, const int32_t* d_ids, int64_t n, float* d_raw, double* d_conf, uint8_t* d_fired,
                        unsigned long long* d_count, cudaStream_t s) {
    const Network& net = h->models[0];
    K2Out o{};
    o.raw = d_raw; o.conf = d_conf; o.fired = d_fired; o.count = d_count; o.trig = net.trig.get();
    if (!h->routed && !net.trig_set) return launch_gru(h, net, stream_k2in(h, d_ids), true, n, o, s);
    TrigTick t{};
    t.ids = d_ids; t.n = n;
    int nt = 0;
    if (net.trig_set) defer_trigger(t, nt, net, 1u, o);
    ProfScope ps(h, 1, s);
    if (h->routed) {
        // NaN fill of the items whose stream lacks bit 0, then the usual kernel with the epilogue's mask.  No list scratch:
        // pb_update_host runs this on three streams at once.
        RouteOut r{};
        r.raw = d_raw; r.conf = d_conf; r.fired = d_fired; r.M = 1;
        route_kernel<<<(int)((n + 255) / 256), 256, 0, s>>>(h->d_route.get(), d_ids, n, r);
        CK(cudaGetLastError());
        if (h->subs[0] == 0) return PB_OK;
        o.route = h->d_route.get(); o.route_bit = 1;
        t.route = h->d_route.get();
    }
    const int rc = launch_gru_kernels(net, h->feat, stream_k2in(h, d_ids), true, n, o, s);
    return rc != PB_OK ? rc : launch_trigger(t, nt, s);
}

PB_API int pb_update(pb_handle* h, const int16_t* d_pcm, const int32_t* d_ids, int64_t n, float* d_raw, double* d_conf,
              uint8_t* d_fired, unsigned long long* d_count, void* stream) {
    int rc = check_tick(h, d_pcm, n);
    if (rc != PB_OK || n == 0) return rc;
    const Network& net = h->models[0];
    if (!net.w) return fail(PB_ERR_STATE, "pb_load_weights has not been called");
    if (!d_conf) return fail(PB_ERR_INVALID, "null d_conf");
    CK(cudaSetDevice(h->cfg.device));
    cudaStream_t s = (cudaStream_t)stream;
    rc = tick_mfcc(h, d_pcm, d_ids, n, s);
    if (rc != PB_OK) return rc;
    return score_model0(h, d_ids, n, d_raw, d_conf, d_fired, d_count, s);
}

// ------------------------------------------------------------------------------------------------
// model bank

// A model's cfg (pb_add_model, pb_pool_load): its front-end fields must equal the handle's.
static int check_front_end(const pb_handle* h, const pb_config& c) {
    if (c.abi_version != PB_ABI_VERSION) return fail(PB_ERR_INVALID, "abi_version %d != %d", c.abi_version, PB_ABI_VERSION);
#define PB_SAME_FRONT_END(f)                                                                                  \
    if (c.f != h->cfg.f)                                                                                      \
        return fail(PB_ERR_INVALID, "front-end field %s = %d differs from the handle's %d: the models of a bank share one MFCC front end", \
                    #f, (int)c.f, (int)h->cfg.f)
    PB_SAME_FRONT_END(sample_rate); PB_SAME_FRONT_END(window_samples); PB_SAME_FRONT_END(hop_samples); PB_SAME_FRONT_END(n_fft);
    PB_SAME_FRONT_END(n_filt); PB_SAME_FRONT_END(n_mfcc); PB_SAME_FRONT_END(n_features); PB_SAME_FRONT_END(use_delta);
    PB_SAME_FRONT_END(vectorizer); PB_SAME_FRONT_END(chunk_samples); PB_SAME_FRONT_END(device);
#undef PB_SAME_FRONT_END
    return PB_OK;
}

PB_API int pb_add_model(pb_handle* h, const pb_config* cfg, const float* kernel, const float* recurrent, const float* bias,
                        const float* dense_w, float dense_b, const double* cd, int64_t cd_len, int32_t* slot) {
    if (!h || !cfg || !kernel || !recurrent || !bias || !dense_w) return fail(PB_ERR_INVALID, "null argument");
    const pb_config& c = *cfg;
    int rc = check_front_end(h, c);
    if (rc != PB_OK) return rc;
    if (h->models.size() >= PB_MAX_MODELS) return fail(PB_ERR_INVALID, "a bank holds at most %d models", PB_MAX_MODELS);
    rc = check_network(c);
    if (rc != PB_OK) return rc;
    CK(cudaSetDevice(c.device));
    // built aside and appended only when complete: a failure leaves the bank as it was
    Network net;
    net.cfg = c;
    net.cfg.max_streams = h->cfg.max_streams;
    build_cdf(net);
    if (cd && cd_len != (int64_t)net.cd.size()) return fail(PB_ERR_INVALID, "cdf length %lld != %zu", (long long)cd_len, net.cd.size());
    if (cd) memcpy(net.cd.data(), cd, cd_len * sizeof(double));
    const cudaError_t e = upload_network_state(net, (size_t)h->cfg.max_streams);
    if (e != cudaSuccess) return fail(PB_ERR_CUDA, "model bank allocation failed: %s", cudaGetErrorString(e));
    rc = load_weights(net, h->feat, kernel, recurrent, bias, dense_w, dense_b);
    if (rc != PB_OK) return rc;
    h->models.push_back(std::move(net));
    if (slot) *slot = (int32_t)h->models.size() - 1;
    return PB_OK;
}

PB_API int pb_num_models(const pb_handle* h) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    return (int)h->models.size();
}

// RING: a tick's bank over the stream ring; otherwise over predict-mode windows (a recorded corpus's frame rows).
template <bool RING>
static int launch_bank(const BankParams& P, int nm, const K2In& in, int64_t n, cudaStream_t s) {
    switch (nm) {
        case 1: return launch_bank_nm<1, RING>(P, in, n, s);
        case 2: return launch_bank_nm<2, RING>(P, in, n, s);
        case 3: return launch_bank_nm<3, RING>(P, in, n, s);
        case 4: return launch_bank_nm<4, RING>(P, in, n, s);
        case 5: return launch_bank_nm<5, RING>(P, in, n, s);
        case 6: return launch_bank_nm<6, RING>(P, in, n, s);
        case 7: return launch_bank_nm<7, RING>(P, in, n, s);
        case 8: return launch_bank_nm<8, RING>(P, in, n, s);
    }
    return fail(PB_ERR_INVALID, "%d fused models", nm);
}

static bool keras_act(const Network& net) {
    return net.cfg.activation == PB_ACT_LINEAR && net.cfg.recurrent_activation == PB_RACT_HARD_SIGMOID;
}

// The network half of a bank tick on a routed handle.  route_kernel writes NaN / NaN / 0 for every unsubscribed (item, model)
// pair and lists the subscribed pairs of each fused model; gru_bank_routed_kernel scans only those (one launch for the models
// with Keras's default activations, one for the others), other networks run their own kernel with the epilogue's mask.  A model
// without subscribers launches nothing.  Grids are sized from the host's subscriber counts: min(n, subs[m]) / 64 tiles each.
static int score_bank_routed(pb_handle* h, const int32_t* d_ids, int64_t n, float* d_raw, double* d_conf, uint8_t* d_fired,
                             unsigned long long* d_count, cudaStream_t s) {
    const int M = (int)h->models.size();
    const K2In in = stream_k2in(h, d_ids);
    const int64_t stride = h->cfg.max_streams;
    int2* lists = h->d_route_list.get();
    unsigned* counts = h->d_route_count.get();
    ProfScope ps(h, 1, s);
    // the lists are the handle's: a routed bank tick on another stream may still be reading them
    CK(cudaStreamWaitEvent(s, h->route_ev, 0));
    CK(cudaMemsetAsync(counts, 0, PB_MAX_MODELS * sizeof(unsigned), s));
    RouteOut r{};
    r.raw = d_raw; r.conf = d_conf; r.fired = d_fired; r.M = M;
    r.lists = lists; r.list_stride = stride; r.count = counts;
    K2Out o[PB_MAX_MODELS];
    TrigTick t{};
    t.route = h->d_route.get(); t.ids = d_ids; t.n = n;
    int nt = 0;
    for (int m = 0; m < M; ++m) {
        o[m] = K2Out{};
        o[m].raw = d_raw ? d_raw + (int64_t)m * n : nullptr;
        o[m].conf = d_conf + (int64_t)m * n;
        o[m].fired = d_fired ? d_fired + (int64_t)m * n : nullptr;
        o[m].count = d_count ? d_count + m : nullptr;
        o[m].trig = h->models[m].trig.get();
        if (h->models[m].trig_set && h->subs[m] > 0) defer_trigger(t, nt, h->models[m], 1u << m, o[m]);
        if (bank_fused(h->models[m], h->feat)) r.listed |= 1u << m;
    }
    route_kernel<<<(int)((n + 255) / 256), 256, 0, s>>>(h->d_route.get(), d_ids, n, r);
    CK(cudaGetLastError());
    for (int m = 0; m < M; ++m) {
        if ((r.listed >> m & 1) || h->subs[m] == 0) continue;
        o[m].route = h->d_route.get();
        o[m].route_bit = 1u << m;
        const int rc = launch_gru_kernels(h->models[m], h->feat, in, true, n, o[m], s);
        if (rc != PB_OK) return rc;
    }
    for (int ka = 0; ka < 2; ++ka) {
        BankParams P{};
        BankRoute R{};
        int tiles = 0;
        for (int m = 0; m < M; ++m) {
            const Network& net = h->models[m];
            if (!(r.listed >> m & 1) || h->subs[m] == 0 || keras_act(net) != (ka == 1)) continue;
            set_bank_slot(P, R.nm, net, o[m]);
            R.list[R.nm] = lists + m * stride;
            R.count[R.nm] = counts + m;
            R.tile0[R.nm++] = tiles;
            tiles += (int)((std::min<int64_t>(n, h->subs[m]) + 63) / 64);
        }
        R.tile0[R.nm] = tiles;
        if (R.nm == 0) continue;
        if (ka) gru_bank_routed_kernel<true><<<tiles, MMA_THREADS, BANK_MODEL_SMEM + BANK_STAGE_SMEM, s>>>(P, R, in);
        else gru_bank_routed_kernel<false><<<tiles, MMA_THREADS, BANK_MODEL_SMEM + BANK_STAGE_SMEM, s>>>(P, R, in);
        CK(cudaGetLastError());
    }
    const int rc = launch_trigger(t, nt, s);
    if (rc != PB_OK) return rc;
    CK(cudaEventRecord(h->route_ev, s));
    return PB_OK;
}

// The network half of a bank tick (pb_update_models, pb_update_ragged): every model scores the windows of the n streams, outputs
// model-major.
static int score_bank(pb_handle* h, const int32_t* d_ids, int64_t n, float* d_raw, double* d_conf, uint8_t* d_fired,
                      unsigned long long* d_count, cudaStream_t s) {
    if (h->routed) return score_bank_routed(h, d_ids, n, d_raw, d_conf, d_fired, d_count, s);
    int rc = PB_OK;
    const int M = (int)h->models.size();
    const K2In in = stream_k2in(h, d_ids);
    ProfScope ps(h, 1, s);
    // the fused family in one gru_bank_kernel launch; other networks one launch each of their own kernel, on the same ring
    BankParams P{};
    TrigTick t{};
    t.ids = d_ids; t.n = n;
    int nm = 0, nt = 0;
    for (int m = 0; m < M; ++m) {
        const Network& net = h->models[m];
        K2Out o{};
        o.raw = d_raw ? d_raw + (int64_t)m * n : nullptr;
        o.conf = d_conf + (int64_t)m * n;
        o.fired = d_fired ? d_fired + (int64_t)m * n : nullptr;
        o.count = d_count ? d_count + m : nullptr;
        o.trig = net.trig.get();
        if (net.trig_set) defer_trigger(t, nt, net, 1u << m, o);
        if (bank_fused(net, h->feat)) {
            set_bank_slot(P, nm++, net, o);
        } else {
            rc = launch_gru_kernels(net, h->feat, in, true, n, o, s);
            if (rc != PB_OK) return rc;
        }
    }
    if (nm) {
        rc = launch_bank<true>(P, nm, in, n, s);
        if (rc != PB_OK) return rc;
    }
    return launch_trigger(t, nt, s);
}

PB_API int pb_update_models(pb_handle* h, const int16_t* d_pcm, const int32_t* d_ids, int64_t n, float* d_raw, double* d_conf,
                            uint8_t* d_fired, unsigned long long* d_count, void* stream) {
    int rc = check_tick(h, d_pcm, n);
    if (rc != PB_OK) return rc;
    if (!h->models[0].w) return fail(PB_ERR_STATE, "pb_load_weights has not been called");
    if (n == 0) return PB_OK;
    if (!d_conf) return fail(PB_ERR_INVALID, "null d_conf");
    CK(cudaSetDevice(h->cfg.device));
    cudaStream_t s = (cudaStream_t)stream;
    rc = tick_mfcc(h, d_pcm, d_ids, n, s);
    if (rc != PB_OK) return rc;
    return score_bank(h, d_ids, n, d_raw, d_conf, d_fired, d_count, s);
}

PB_API int pb_update_ragged(pb_handle* h, const int16_t* d_pcm, const int64_t* d_offsets, int64_t max_len, const int32_t* d_ids,
                            int64_t n, float* d_raw, double* d_conf, uint8_t* d_fired, unsigned long long* d_count, void* stream) {
    int rc = check_tick(h, d_pcm, n);
    if (rc != PB_OK) return rc;
    if (!d_offsets) return fail(PB_ERR_INVALID, "null d_offsets");
    if (!d_conf) return fail(PB_ERR_INVALID, "null d_conf");
    if (max_len < 1) return fail(PB_ERR_INVALID, "max_len = %lld must be >= 1", (long long)max_len);
    if (!h->models[0].w) return fail(PB_ERR_STATE, "pb_load_weights has not been called");
    if (h->k1_mode != 0) return fail(PB_ERR_STATE, "ragged ticks run only with k1 mode 0");
    if (n == 0) return PB_OK;
    CK(cudaSetDevice(h->cfg.device));
    cudaStream_t s = (cudaStream_t)stream;
    h->ragged = true;
    rc = append_history(h, d_pcm, d_offsets, max_len, d_ids, n, s);
    if (rc != PB_OK) return rc;
    rc = launch_ragged_mfcc(h, d_pcm, d_offsets, max_len, d_ids, n, s);
    if (rc != PB_OK) return rc;
    // one model: pb_update's network path, so a ragged tick of uniform chunks equals pb_update bit for bit; a bank:
    // pb_update_models's
    if (h->models.size() == 1) return score_model0(h, d_ids, n, d_raw, d_conf, d_fired, d_count, s);
    return score_bank(h, d_ids, n, d_raw, d_conf, d_fired, d_count, s);
}

// ------------------------------------------------------------------------------------------------
// recorded corpora (corpus.cuh)

// Frames vectorize_raw yields for n samples under front end c (pb_mfcc_frames without a handle).
static int64_t corpus_frames(const pb_config& c, int64_t n) {
    const int64_t rel = c.window_samples + (c.vectorizer == PB_VEC_SPEECHPY_MFCCS ? c.hop_samples : 0);
    return n < rel ? 0 : (n - rel) / c.hop_samples + 1;
}

static int check_corpus_schedule(const pb_config& c, int32_t schedule, int64_t chunk) {
    if (schedule != PB_CORPUS_LISTENER && schedule != PB_CORPUS_SIMULATE) return fail(PB_ERR_INVALID, "unknown corpus schedule %d", schedule);
    if (chunk < 1) return fail(PB_ERR_INVALID, "chunk = %lld must be >= 1", (long long)chunk);
    if (schedule == PB_CORPUS_SIMULATE && chunk / c.hop_samples < 1)
        return fail(PB_ERR_INVALID, "simulate chunk %lld is shorter than one hop (%d samples)", (long long)chunk, c.hop_samples);
    return PB_OK;
}

// Windows of one recording of n samples (arguments checked).  LISTENER: one per complete chunk.  SIMULATE:
// len(range(n_features, n_frames, chunk // hop)) (simulate.py:96-99).
static int64_t corpus_windows(const pb_config& c, int32_t schedule, int64_t chunk, int64_t n) {
    if (schedule == PB_CORPUS_LISTENER) return n / chunk;
    const int64_t nf = corpus_frames(c, n), hops = chunk / c.hop_samples;
    return nf > c.n_features ? (nf - c.n_features + hops - 1) / hops : 0;
}

PB_API int64_t pb_corpus_windows(const pb_config* cfg, int32_t schedule, int64_t chunk, int64_t n_samples) {
    if (!cfg) return fail(PB_ERR_INVALID, "cfg is null");
    if (cfg->window_samples < 1 || cfg->hop_samples < 1 || cfg->n_features < 1)
        return fail(PB_ERR_INVALID, "window_samples, hop_samples and n_features must be positive");
    if (n_samples < 0) return fail(PB_ERR_INVALID, "n_samples = %lld is negative", (long long)n_samples);
    const int rc = check_corpus_schedule(*cfg, schedule, chunk);
    return rc != PB_OK ? rc : corpus_windows(*cfg, schedule, chunk, n_samples);
}

// Grows a workspace array to n elements.  The replaced array is freed only after the previous corpus call is done with it.
template <typename T>
static cudaError_t corpus_grow(const DevArray<T>& a, size_t n, DevArray<T>& fresh) {
    if (a.size() >= n) return cudaSuccess;
    return fresh.alloc(n + n / 4);
}

// The checks every corpus call shares (pb_score_corpus, pb_score_corpus_pool); raw_required: d_raw may not be null.
static int check_corpus(const pb_handle* h, const int16_t* d_pcm, const int64_t* h_offsets, int64_t n_rec, int32_t divisor,
                        int32_t schedule, int64_t chunk, const float* d_raw, bool raw_required, const int64_t* d_above,
                        const double* d_sum) {
    const pb_config& c = h->cfg;
    if (n_rec < 0 || n_rec > INT32_MAX) return fail(PB_ERR_INVALID, "n_rec = %lld outside [0, 2^31)", (long long)n_rec);
    if (!h_offsets) return fail(PB_ERR_INVALID, "null h_offsets");
    if (raw_required && !d_raw) return fail(PB_ERR_INVALID, "null d_raw");
    if (divisor != 32768 && divisor != 32767) return fail(PB_ERR_INVALID, "divisor %d: 32768 (buffer_to_audio) or 32767 (load_audio)", divisor);
    const int rc = check_corpus_schedule(c, schedule, chunk);
    if (rc != PB_OK) return rc;
    if (schedule == PB_CORPUS_LISTENER && (d_above || d_sum)) return fail(PB_ERR_INVALID, "d_above and d_sum belong to the simulate schedule");
    if (h_offsets[0] < 0) return fail(PB_ERR_INVALID, "offset 0 = %lld is negative", (long long)h_offsets[0]);
    for (int64_t r = 0; r < n_rec; ++r)
        if (h_offsets[r + 1] < h_offsets[r]) return fail(PB_ERR_INVALID, "offsets decrease at recording %lld", (long long)r);
    if (h_offsets[n_rec] > h_offsets[0] && !d_pcm) return fail(PB_ERR_INVALID, "null d_pcm");
    return PB_OK;
}

// K1's host plan of a corpus call: window prefix, frame rows, and the recordings in pair-list order (aligned geometry first).
struct CorpusPlan {
    std::vector<long long> win0, frow;
    std::vector<long long> starts;   // labelled clips: the window table itself, one window per recording
    std::vector<CorpusRec> recs;
    long long rows = 1, n_fast_pairs = 0, n_pairs = 0, W = 0;
};

// crop > 0 (labelled clips, vectorization.py:73-82): each recording is its last `crop` samples, framed from the first of
// them, and has one window, the n_features rows ending at its last frame (row 0's zeros when it has no frame).
static CorpusPlan corpus_plan(const pb_handle* h, const int16_t* d_pcm, const int64_t* h_offsets, int64_t n_rec, int32_t schedule,
                              int64_t chunk, int64_t crop = 0) {
    const pb_config& c = h->cfg;
    const int T = c.n_features;
    const bool fast = h->fast_ok && !h->force_generic && (uintptr_t)d_pcm % 16 == 0;
    CorpusPlan p;
    p.win0.resize((size_t)n_rec + 1);
    p.frow.resize((size_t)n_rec);
    p.recs.reserve((size_t)n_rec + 1);
    p.win0[0] = 0;
    if (crop > 0) p.starts.resize((size_t)n_rec);
    for (int pass = 0; pass < 2; ++pass)
        for (int64_t r = 0; r < n_rec; ++r) {
            const int64_t len = h_offsets[r + 1] - h_offsets[r], L = crop > 0 ? std::min(len, crop) : len;
            const int64_t src = h_offsets[r] + len - L, nf = corpus_frames(c, L);
            const bool fr = fast && src % 8 == 0;
            if (pass == 0) {
                p.win0[r + 1] = p.win0[r] + (crop > 0 ? 1 : corpus_windows(c, schedule, chunk, L));
                p.frow[r] = p.rows + T - 1;
                p.rows += T - 1 + nf;
                if (crop > 0) p.starts[r] = nf ? p.frow[r] + nf - T : 0;
            }
            if (fr != (pass == 0)) continue;
            p.recs.push_back(CorpusRec{src, p.frow[r], nf, p.n_pairs});
            p.n_pairs += (nf + 1) / 2;
            if (fr) p.n_fast_pairs = p.n_pairs;
        }
    p.recs.push_back(CorpusRec{0, 0, 0, p.n_pairs});
    p.W = p.win0[n_rec];
    return p;
}

// Sizes of pb_score_corpus_pool's and pb_score_corpus_pairs's own workspace arrays (0 for pb_score_corpus).
struct CorpusPoolSizes {
    size_t groups = 0, ids = 0, raw = 0;
    size_t pairs = 0, pw0 = 0, starts = 0, tiles = 0;
    size_t thr = 0, targets = 0;     // pb_score_dataset
};

// Grows the workspace for plan p, all at once, so that a failed allocation leaves the handle as it was; then orders s after
// the previous corpus call.
static int corpus_reserve(pb_handle* h, const CorpusPlan& p, int64_t n_rec, const CorpusPoolSizes& ps, cudaStream_t s) {
    if (!h->corpus_ev) CK(cudaEventCreateWithFlags(&h->corpus_ev, cudaEventDisableTiming));
    DevArray<float> f_rows, f_raw; DevArray<CorpusPair> f_pairs; DevArray<long long> f_starts, f_win0, f_frow; DevArray<CorpusRec> f_recs;
    DevArray<int2> f_groups; DevArray<int> f_ids;
    DevArray<int2> f_ppairs; DevArray<long long> f_pw0, f_pstarts; DevArray<PairTile> f_tiles;
    DevArray<float> f_thr; DevArray<uint8_t> f_targets;
    cudaError_t e = corpus_grow(h->d_cw_rows, (size_t)p.rows * h->row_stride, f_rows);
    if (e == cudaSuccess) e = corpus_grow(h->d_cw_pairs, (size_t)p.n_pairs, f_pairs);
    if (e == cudaSuccess) e = corpus_grow(h->d_cw_starts, (size_t)p.W, f_starts);
    if (e == cudaSuccess) e = corpus_grow(h->d_cw_win0, (size_t)n_rec + 1, f_win0);
    if (e == cudaSuccess) e = corpus_grow(h->d_cw_frow, (size_t)n_rec, f_frow);
    if (e == cudaSuccess) e = corpus_grow(h->d_cw_recs, p.recs.size(), f_recs);
    if (e == cudaSuccess) e = corpus_grow(h->d_cp_groups, ps.groups, f_groups);
    if (e == cudaSuccess) e = corpus_grow(h->d_cp_ids, ps.ids, f_ids);
    if (e == cudaSuccess && h->d_cp_raw.size() < ps.raw) e = f_raw.alloc(ps.raw);     // capped: no headroom
    if (e == cudaSuccess) e = corpus_grow(h->d_pp_pairs, ps.pairs, f_ppairs);
    if (e == cudaSuccess) e = corpus_grow(h->d_pp_pw0, ps.pw0, f_pw0);
    if (e == cudaSuccess && h->d_pp_starts.size() < ps.starts) e = f_pstarts.alloc(ps.starts);   // capped: no headroom
    if (e == cudaSuccess) e = corpus_grow(h->d_pp_tiles, ps.tiles, f_tiles);
    if (e == cudaSuccess) e = corpus_grow(h->d_ds_thr, ps.thr, f_thr);
    if (e == cudaSuccess) e = corpus_grow(h->d_ds_targets, ps.targets, f_targets);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(PB_ERR_CUDA, "corpus workspace allocation failed (%lld frame rows, %lld windows): %s", p.rows, p.W, cudaGetErrorString(e));
    }
    const bool grows = f_rows.get() || f_pairs.get() || f_starts.get() || f_win0.get() || f_frow.get() || f_recs.get() ||
                       f_groups.get() || f_ids.get() || f_raw.get() || f_ppairs.get() || f_pw0.get() || f_pstarts.get() ||
                       f_tiles.get() || f_thr.get() || f_targets.get();
    if (grows) CK(cudaEventSynchronize(h->corpus_ev));            // the previous call may still read what is replaced
    if (f_rows.get()) h->d_cw_rows = std::move(f_rows);
    if (f_pairs.get()) h->d_cw_pairs = std::move(f_pairs);
    if (f_starts.get()) h->d_cw_starts = std::move(f_starts);
    if (f_win0.get()) h->d_cw_win0 = std::move(f_win0);
    if (f_frow.get()) h->d_cw_frow = std::move(f_frow);
    if (f_recs.get()) h->d_cw_recs = std::move(f_recs);
    if (f_groups.get()) h->d_cp_groups = std::move(f_groups);
    if (f_ids.get()) h->d_cp_ids = std::move(f_ids);
    if (f_raw.get()) h->d_cp_raw = std::move(f_raw);
    if (f_ppairs.get()) h->d_pp_pairs = std::move(f_ppairs);
    if (f_pw0.get()) h->d_pp_pw0 = std::move(f_pw0);
    if (f_pstarts.get()) h->d_pp_starts = std::move(f_pstarts);
    if (f_tiles.get()) h->d_pp_tiles = std::move(f_tiles);
    if (f_thr.get()) h->d_ds_thr = std::move(f_thr);
    if (f_targets.get()) h->d_ds_targets = std::move(f_targets);
    CK(cudaStreamWaitEvent(s, h->corpus_ev, 0));                      // a corpus call on another stream may still use it
    return PB_OK;
}

// K1 of a corpus call: the plan's device copies, the frame buffer and the window table (profile slot 0).
static int corpus_k1(pb_handle* h, const CorpusPlan& p, const int16_t* d_pcm, int64_t n_rec, int32_t divisor, int32_t schedule,
                     int64_t chunk, cudaStream_t s) {
    const pb_config& c = h->cfg;
    CK(cudaMemcpyAsync(h->d_cw_win0.get(), p.win0.data(), p.win0.size() * sizeof(long long), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(h->d_cw_frow.get(), p.frow.data(), p.frow.size() * sizeof(long long), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(h->d_cw_recs.get(), p.recs.data(), p.recs.size() * sizeof(CorpusRec), cudaMemcpyHostToDevice, s));
    if (p.n_pairs == 0 && p.W == 0) return PB_OK;
    float* frames = h->d_cw_rows.get();
    ProfScope ps(h, 0, s);
    CK(cudaMemsetAsync(frames, 0, (size_t)p.rows * h->row_stride * sizeof(float), s));
    const float inv = 1.0f / (float)divisor, scale = inv * inv / (float)c.n_fft;
    if (p.n_pairs > 0) {
        corpus_pairs_kernel<<<(unsigned)((p.n_pairs + 255) / 256), 256, 0, s>>>(h->d_cw_recs.get(), (int)p.recs.size() - 1, p.n_pairs,
                                                                              c.hop_samples, h->d_cw_pairs.get());
        CK(cudaGetLastError());
    }
    if (p.n_fast_pairs > 0) {
        const int grid = (int)std::min<int64_t>((p.n_fast_pairs + K1F_WARPS - 1) / K1F_WARPS, (int64_t)h->sm_count * 4);
        mfcc_fast_corpus_kernel<<<grid, K1F_THREADS, h->k1_fast_smem, s>>>(d_pcm, h->d_cw_pairs.get(), p.n_fast_pairs, c.hop_samples, scale,
                                                                          mel_tables(h), fast_tables(h), frames, h->row_stride);
        CK(cudaGetLastError());
    }
    if (p.n_pairs > p.n_fast_pairs) {
        const int64_t tiles = (p.n_pairs - p.n_fast_pairs + K1_TILE / 2 - 1) / (K1_TILE / 2);
        const int grid = (int)std::min<int64_t>(tiles, (int64_t)h->sm_count * 4);
        mfcc_corpus_kernel<<<grid, K1_THREADS, h->k1_batch_smem, s>>>(d_pcm, h->d_cw_pairs.get() + p.n_fast_pairs, p.n_pairs - p.n_fast_pairs,
                                                                     c.hop_samples, h->used, scale, mel_tables(h), frames, h->row_stride);
        CK(cudaGetLastError());
    }
    if (!p.starts.empty()) {
        CK(cudaMemcpyAsync(h->d_cw_starts.get(), p.starts.data(), p.starts.size() * sizeof(long long), cudaMemcpyHostToDevice, s));
    } else if (p.W > 0) {
        corpus_windows_kernel<<<(unsigned)((p.W + 255) / 256), 256, 0, s>>>(h->d_cw_win0.get(), h->d_cw_frow.get(), (int)n_rec, p.W, schedule, chunk,
                                                                          h->rel_window, c.hop_samples, c.n_features, h->d_cw_starts.get());
        CK(cudaGetLastError());
    }
    return PB_OK;
}

// Predict-mode input of a corpus call's scans: the windows in place in the frame buffer.
static K2In corpus_k2in(const pb_handle* h) {
    K2In in{};
    in.inputs = h->d_cw_rows.get(); in.starts = h->d_cw_starts.get(); in.row_stride = h->row_stride;
    in.T = h->cfg.n_features; in.F_base = h->n_out; in.use_delta = h->cfg.use_delta;
    return in;
}

// The trigger pass's fields shared by every row.
static CorpusTrig corpus_trig(const pb_handle* h, int64_t n_rec, int64_t W, int32_t schedule, int64_t chunk, double threshold) {
    CorpusTrig t{};
    t.win0 = h->d_cw_win0.get(); t.W = W; t.n_rec = (int)n_rec; t.schedule = schedule;
    t.hot_f = (float)(1.0 - threshold); t.above_f = (float)threshold;
    t.sim_reset = trigger_reset(chunk);
    return t;
}

// Records corpus_ev after the call's work, even when a launch failed, so the next call orders itself after whatever this
// one queued.
static int corpus_done(pb_handle* h, cudaStream_t s, int rc) {
    const cudaError_t er = cudaEventRecord(h->corpus_ev, s);
    if (rc != PB_OK) return rc;
    if (er != cudaSuccess) return fail(PB_ERR_CUDA, "cudaEventRecord failed: %s", cudaGetErrorString(er));
    return PB_OK;
}

PB_API int pb_score_corpus(pb_handle* h, const int16_t* d_pcm, const int64_t* h_offsets, int64_t n_rec, int32_t divisor,
                           int32_t schedule, int64_t chunk, double threshold, float* d_raw, double* d_conf, uint8_t* d_fired,
                           int64_t* d_activations, int64_t* d_above, double* d_sum, void* stream) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    int rc = check_corpus(h, d_pcm, h_offsets, n_rec, divisor, schedule, chunk, d_raw, true, d_above, d_sum);
    if (rc != PB_OK) return rc;
    if (!h->models[0].w) return fail(PB_ERR_STATE, "pb_load_weights has not been called");
    if (n_rec == 0) return PB_OK;
    CK(cudaSetDevice(h->cfg.device));
    cudaStream_t s = (cudaStream_t)stream;
    const int M = (int)h->models.size();
    const CorpusPlan p = corpus_plan(h, d_pcm, h_offsets, n_rec, schedule, chunk);
    const long long W = p.W;
    rc = corpus_reserve(h, p, n_rec, CorpusPoolSizes{}, s);
    if (rc != PB_OK) return rc;
    auto launch = [&]() -> int {
        rc = corpus_k1(h, p, d_pcm, n_rec, divisor, schedule, chunk, s);
        if (rc != PB_OK) return rc;
        ProfScope ps(h, 1, s);
        if (W > 0) {
            // every model scans the windows in place.  One model runs pb_predict's dispatch (the warp-per-window kernel up to
            // 8 192 windows for the default network); a bank runs its fused family in one predict-mode bank launch, the others
            // one launch each
            const K2In in = corpus_k2in(h);
            BankParams P{};
            int nm = 0;
            for (int m = 0; m < M; ++m) {
                const Network& net = h->models[m];
                K2Out o{};
                o.raw = d_raw + (int64_t)m * W;
                o.conf = d_conf ? d_conf + (int64_t)m * W : nullptr;
                if (M > 1 && bank_fused(net, h->feat)) {
                    set_bank_slot(P, nm++, net, o);
                } else {
                    rc = launch_gru_kernels(net, h->feat, in, false, W, o, s);
                    if (rc != PB_OK) return rc;
                }
            }
            if (nm) {
                rc = launch_bank<false>(P, nm, in, W, s);
                if (rc != PB_OK) return rc;
            }
        }
        if (d_fired || d_activations || d_above || d_sum) {
            CorpusTrig t = corpus_trig(h, n_rec, W, schedule, chunk, threshold);
            t.raw = d_raw; t.conf = d_conf; t.fired = d_fired; t.activations = d_activations; t.above = d_above; t.sum = d_sum;
            CorpusBankDP dp{};
            for (int m = 0; m < M; ++m) {
                dp.dp[m] = decode_params(h->models[m]);
                dp.dp[m].trigger_reset = trigger_reset(2 * chunk);            // TriggerDetector(2c bytes, ...) of a chunk-c listener
            }
            const unsigned per = CORPUS_TRIG_THREADS / 32;
            corpus_trigger_kernel<<<dim3((unsigned)((n_rec + per - 1) / per), (unsigned)M), CORPUS_TRIG_THREADS, 0, s>>>(t, dp);
            CK(cudaGetLastError());
        }
        return PB_OK;
    };
    return corpus_done(h, s, launch());
}

// ------------------------------------------------------------------------------------------------
// pool models over a recorded corpus (corpus_pool.cuh)

// Bytes of raw a pb_score_corpus_pool call without d_raw keeps on the device for its trigger pass: rows are scanned in
// batches of max(1, cap / (4 W)) models.
constexpr int64_t CORPUS_POOL_RAW_CAP = 256ll << 20;
// Models per group and grid order of the scan (DESIGN §6, "Pool models over a recorded corpus"); pb_debug_corpus_pool_scan
// picks others for A/B timing.
constexpr int CORPUS_POOL_NM = 1;
constexpr int CORPUS_POOL_GROUPS_FAST = 1;

template <int NM, bool KERAS_ACT>
static int launch_pool_corpus(PoolCorpus c, const K2In& in, cudaStream_t s) {
    constexpr size_t smem = (size_t)NM * BANK_MODEL_SMEM;
    if constexpr (smem > 48 * 1024) CK(ensure_dyn_smem(pool_corpus_kernel<NM, KERAS_ACT>, smem));
    const int64_t total = c.n_groups * c.n_tiles;
    if (total == 0) return PB_OK;
    const int64_t gx = std::min<int64_t>(total, 1ll << 30), gy = (total + gx - 1) / gx;
    pool_corpus_kernel<NM, KERAS_ACT><<<dim3((unsigned)gx, (unsigned)gy), MMA_THREADS, smem, s>>>(c, in);
    CK(cudaGetLastError());
    return PB_OK;
}

static int launch_pool_corpus_nm(int nm, bool keras, const PoolCorpus& c, const K2In& in, cudaStream_t s) {
    switch (nm) {
        case 1: return keras ? launch_pool_corpus<1, true>(c, in, s) : launch_pool_corpus<1, false>(c, in, s);
        case 2: return keras ? launch_pool_corpus<2, true>(c, in, s) : launch_pool_corpus<2, false>(c, in, s);
        case 4: return launch_pool_corpus<4, false>(c, in, s);
        case 8: return launch_pool_corpus<8, false>(c, in, s);
    }
    return fail(PB_ERR_INVALID, "%d models per group", nm);
}

// The scan's groups of k requested models in batches of `rows`: within a batch, per activation class (Keras's defaults first
// where they are compiled in), NM requested rows each in request order, a partial last group padded with row -1.  Batch b,
// class ka: groups [g0[2b + ka], g0[2b + ka + 1]).
static void pool_corpus_groups(const pb_handle* h, const int32_t* h_model_ids, int64_t k, int64_t rows, int NM,
                               std::vector<int2>& groups, std::vector<int64_t>& g0) {
    const bool split = pool_corpus_keras(NM);
    const int64_t n_batches = (k + rows - 1) / rows;
    g0.assign((size_t)n_batches * 2 + 1, 0);
    for (int64_t b = 0; b < n_batches; ++b) {
        const int64_t b0 = b * rows, b1 = std::min<int64_t>(k, b0 + rows);
        for (int ka = 0; ka < 2; ++ka) {
            g0[2 * b + ka] = (int64_t)groups.size() / NM;
            int at = 0;
            for (int64_t i = b0; i < b1; ++i) {
                if ((split ? h->pool_keras[h_model_ids[i]] : 1) != ka) continue;
                groups.push_back(make_int2(h_model_ids[i], (int)(i - b0)));
                at = (at + 1) % NM;
            }
            for (const int2 first = at ? groups[groups.size() - at] : int2{}; at && at < NM; ++at)
                groups.push_back(make_int2(first.x, -1));
        }
    }
    g0[2 * n_batches] = (int64_t)groups.size() / NM;
}

PB_API int pb_debug_corpus_pool_rows(pb_handle* h, int64_t rows) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    if (rows < 0) return fail(PB_ERR_INVALID, "rows = %lld is negative", (long long)rows);
    h->corpus_pool_rows = rows;
    return PB_OK;
}

PB_API int pb_debug_corpus_pool_scan(pb_handle* h, int32_t nm, int32_t groups_fast) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    if (nm != 0 && nm != 1 && nm != 2 && nm != 4 && nm != 8) return fail(PB_ERR_INVALID, "nm = %d: 0 (default), 1, 2, 4 or 8", nm);
    if (groups_fast < -1 || groups_fast > 1) return fail(PB_ERR_INVALID, "groups_fast = %d: -1 (default), 0 or 1", groups_fast);
    h->corpus_pool_nm = nm;
    h->corpus_pool_order = groups_fast;
    return PB_OK;
}

PB_API int pb_score_corpus_pool(pb_handle* h, const int16_t* d_pcm, const int64_t* h_offsets, int64_t n_rec,
                                const int32_t* h_model_ids, int64_t k, int32_t divisor, int32_t schedule, int64_t chunk,
                                double threshold, float* d_raw, double* d_conf, uint8_t* d_fired, int64_t* d_activations,
                                int64_t* d_above, double* d_sum, void* stream) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    int rc = check_corpus(h, d_pcm, h_offsets, n_rec, divisor, schedule, chunk, d_raw, false, d_above, d_sum);
    if (rc != PB_OK) return rc;
    const bool reduce = d_fired || d_activations || d_above || d_sum;
    if (!d_raw && !d_conf && !reduce) return fail(PB_ERR_INVALID, "every output is null");
    if (!h->pool) return fail(PB_ERR_STATE, "no model pool: call pb_set_pool first");
    if (k < 0) return fail(PB_ERR_INVALID, "k = %lld is negative", (long long)k);
    if (k > 0 && !h_model_ids) return fail(PB_ERR_INVALID, "null h_model_ids");
    for (int64_t i = 0; i < k; ++i) {
        const int32_t m = h_model_ids[i];
        if (m < 0 || m >= h->pool_models)
            return fail(PB_ERR_INVALID, "model id %d (entry %lld) outside [0, max_models = %d)", m, (long long)i, h->pool_models);
        if (h->pool_cd_of[m] == h->pool_cd.end())
            return fail(PB_ERR_INVALID, "pool slot %d (entry %lld) holds no model: pb_pool_load it first", m, (long long)i);
    }
    if (n_rec == 0 || k == 0) return PB_OK;
    CK(cudaSetDevice(h->cfg.device));
    cudaStream_t s = (cudaStream_t)stream;
    const CorpusPlan p = corpus_plan(h, d_pcm, h_offsets, n_rec, schedule, chunk);
    const long long W = p.W;
    // rows per batch: all of them when the caller's d_raw holds raw (or no trigger pass needs it), else as many as the cap holds
    const bool own_raw = !d_raw && reduce && W > 0;
    int64_t rows = k;
    if (own_raw) {
        rows = std::max<int64_t>(1, CORPUS_POOL_RAW_CAP / (4 * W));
        if (h->corpus_pool_rows > 0) rows = std::min<int64_t>(rows, h->corpus_pool_rows);
        rows = std::min<int64_t>(rows, k);
    }
    const int NM = h->corpus_pool_nm ? h->corpus_pool_nm : CORPUS_POOL_NM;
    const bool split = pool_corpus_keras(NM);
    const int64_t n_batches = (k + rows - 1) / rows;
    std::vector<int2> groups;
    std::vector<int64_t> g0;
    pool_corpus_groups(h, h_model_ids, k, rows, NM, groups, g0);
    CorpusPoolSizes ps;
    ps.groups = groups.size();
    ps.ids = (size_t)k;
    ps.raw = own_raw ? (size_t)(rows * W) : 0;
    rc = corpus_reserve(h, p, n_rec, ps, s);
    if (rc != PB_OK) return rc;
    const int order = h->corpus_pool_order >= 0 ? h->corpus_pool_order : CORPUS_POOL_GROUPS_FAST;
    auto launch = [&]() -> int {
        rc = corpus_k1(h, p, d_pcm, n_rec, divisor, schedule, chunk, s);
        if (rc != PB_OK) return rc;
        if (W == 0 && !reduce) return PB_OK;
        CK(cudaMemcpyAsync(h->d_cp_groups.get(), groups.data(), groups.size() * sizeof(int2), cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(h->d_cp_ids.get(), h_model_ids, (size_t)k * sizeof(int32_t), cudaMemcpyHostToDevice, s));
        ProfScope ps(h, 1, s);
        const K2In in = corpus_k2in(h);
        for (int64_t b = 0; b < n_batches; ++b) {
            const int64_t b0 = b * rows, nb = std::min<int64_t>(k, b0 + rows) - b0;
            float* raw = own_raw ? h->d_cp_raw.get() : d_raw ? d_raw + b0 * W : nullptr;
            if (W > 0) {
                PoolCorpus c{};
                c.slots = h->d_pool_slots.get(); c.n_tiles = (W + 63) / 64; c.raw = raw;
                c.conf = d_conf ? d_conf + b0 * W : nullptr; c.W = W; c.groups_fast = order;
                for (int ka = 0; ka < 2; ++ka) {
                    c.groups = h->d_cp_groups.get() + g0[2 * b + ka] * NM;
                    c.n_groups = g0[2 * b + ka + 1] - g0[2 * b + ka];
                    rc = launch_pool_corpus_nm(NM, split && ka == 1, c, in, s);
                    if (rc != PB_OK) return rc;
                }
            }
            if (!reduce) continue;
            // rows b0 .. b0 + nb - 1, at most 65 535 per launch (gridDim.y)
            for (int64_t y0 = 0; y0 < nb; y0 += 65535) {
                const int64_t r0 = b0 + y0, ny = std::min<int64_t>(65535, nb - y0);
                CorpusTrig t = corpus_trig(h, n_rec, W, schedule, chunk, threshold);
                t.raw = raw ? raw + y0 * W : nullptr;
                t.conf = d_conf ? d_conf + r0 * W : nullptr;
                t.fired = d_fired ? d_fired + r0 * W : nullptr;
                t.activations = d_activations ? d_activations + r0 * n_rec : nullptr;
                t.above = d_above ? d_above + r0 * n_rec : nullptr;
                t.sum = d_sum ? d_sum + r0 * n_rec : nullptr;
                CorpusPoolDP dp{h->d_pool_slots.get(), h->d_cp_ids.get() + r0, trigger_reset(2 * chunk)};
                const unsigned per = CORPUS_TRIG_THREADS / 32;
                corpus_trigger_kernel<<<dim3((unsigned)((n_rec + per - 1) / per), (unsigned)ny), CORPUS_TRIG_THREADS, 0, s>>>(t, dp);
                CK(cudaGetLastError());
            }
        }
        return PB_OK;
    };
    return corpus_done(h, s, launch());
}

// ------------------------------------------------------------------------------------------------
// pool models over chosen recordings (corpus_pairs.cuh)

// Pair-windows per batch: the batch's window table takes 8 B per pair-window (256 MB), its raw without d_raw 4 B.
constexpr int64_t CORPUS_PAIRS_BATCH = 1ll << 25;

template <bool KERAS_ACT>
static int launch_pairs_corpus(const PairsCorpus& c, const K2In& in, cudaStream_t s) {
    if (c.n_tiles == 0) return PB_OK;
    const int64_t gx = std::min<int64_t>(c.n_tiles, 1ll << 30), gy = (c.n_tiles + gx - 1) / gx;
    pairs_corpus_kernel<KERAS_ACT><<<dim3((unsigned)gx, (unsigned)gy), MMA_THREADS, BANK_MODEL_SMEM, s>>>(c, in);
    CK(cudaGetLastError());
    return PB_OK;
}

// Scan tiles of pairs p0 .. p1 - 1 (pool slot, recording), pair p's windows at P[p] .. P[p + 1] - 1: tiles of 64 pair-windows
// within each run of one model, batch-local, the Keras-activation class first.  Returns that class's tile count.
static int64_t pair_tiles(const pb_handle* h, const std::vector<int2>& pairs, const std::vector<long long>& P, int64_t p0,
                          int64_t p1, std::vector<PairTile>& tiles) {
    tiles.clear();
    int64_t n_keras = 0;
    for (int ka = 1; ka >= 0; --ka) {
        for (int64_t a = p0; a < p1;) {
            int64_t e = a + 1;
            while (e < p1 && pairs[e].x == pairs[a].x) ++e;
            if (h->pool_keras[pairs[a].x] == ka)
                for (long long q = P[a]; q < P[e]; q += 64)
                    tiles.push_back(PairTile{q - P[p0], pairs[a].x, (int)std::min<long long>(64, P[e] - q)});
            a = e;
        }
        if (ka == 1) n_keras = (int64_t)tiles.size();
    }
    return n_keras;
}

PB_API int pb_debug_corpus_pairs_batch(pb_handle* h, int64_t windows) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    if (windows < 0) return fail(PB_ERR_INVALID, "windows = %lld is negative", (long long)windows);
    h->corpus_pairs_batch = windows;
    return PB_OK;
}

PB_API int pb_score_corpus_pairs(pb_handle* h, const int16_t* d_pcm, const int64_t* h_offsets, int64_t n_rec,
                                 const int32_t* h_pair_models, const int32_t* h_pair_recs, int64_t n_pairs,
                                 int32_t divisor, int32_t schedule, int64_t chunk, double threshold,
                                 float* d_raw, double* d_conf, uint8_t* d_fired,
                                 int64_t* d_activations, int64_t* d_above, double* d_sum,
                                 double hit_threshold, int64_t* d_hits, int64_t hit_capacity,
                                 unsigned long long* d_n_hits, void* stream) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    int rc = check_corpus(h, d_pcm, h_offsets, n_rec, divisor, schedule, chunk, d_raw, false, d_above, d_sum);
    if (rc != PB_OK) return rc;
    const bool reduce = d_fired || d_activations || d_above || d_sum, hits = d_n_hits != nullptr;
    if (!d_raw && !d_conf && !reduce && !hits) return fail(PB_ERR_INVALID, "every output is null");
    if (!h->pool) return fail(PB_ERR_STATE, "no model pool: call pb_set_pool first");
    if (n_pairs < 0 || n_pairs > INT32_MAX) return fail(PB_ERR_INVALID, "n_pairs = %lld outside [0, 2^31)", (long long)n_pairs);
    if (n_pairs > 0 && (!h_pair_models || !h_pair_recs)) return fail(PB_ERR_INVALID, "null h_pair_models or h_pair_recs");
    for (int64_t i = 0; i < n_pairs; ++i) {
        const int32_t m = h_pair_models[i], r = h_pair_recs[i];
        if (m < 0 || m >= h->pool_models)
            return fail(PB_ERR_INVALID, "model id %d (pair %lld) outside [0, max_models = %d)", m, (long long)i, h->pool_models);
        if (h->pool_cd_of[m] == h->pool_cd.end())
            return fail(PB_ERR_INVALID, "pool slot %d (pair %lld) holds no model: pb_pool_load it first", m, (long long)i);
        if (r < 0 || r >= n_rec)
            return fail(PB_ERR_INVALID, "recording id %d (pair %lld) outside [0, n_rec = %lld)", r, (long long)i, (long long)n_rec);
    }
    if (hit_capacity < 0) return fail(PB_ERR_INVALID, "hit_capacity = %lld is negative", (long long)hit_capacity);
    if (hit_capacity > 0 && !d_hits) return fail(PB_ERR_INVALID, "null d_hits with hit_capacity = %lld", (long long)hit_capacity);
    if (d_hits && !hits) return fail(PB_ERR_INVALID, "d_hits without d_n_hits");
    if (hits && schedule == PB_CORPUS_SIMULATE) return fail(PB_ERR_INVALID, "hits belong to the listener schedule");
    CK(cudaSetDevice(h->cfg.device));
    cudaStream_t s = (cudaStream_t)stream;
    if (n_pairs == 0) {
        if (hits) CK(cudaMemsetAsync(d_n_hits, 0, sizeof(unsigned long long), s));
        return PB_OK;
    }
    const CorpusPlan plan = corpus_plan(h, d_pcm, h_offsets, n_rec, schedule, chunk);
    // pair p's windows are P[p] .. P[p + 1] - 1 of every per-window output
    std::vector<long long> P((size_t)n_pairs + 1);
    std::vector<int2> pairs((size_t)n_pairs);
    P[0] = 0;
    for (int64_t i = 0; i < n_pairs; ++i) {
        const int r = h_pair_recs[i];
        P[i + 1] = P[i] + (plan.win0[r + 1] - plan.win0[r]);
        pairs[i] = make_int2(h_pair_models[i], r);
    }
    // batches of consecutive pairs, bp[b] .. bp[b + 1] - 1, of at most `cap` pair-windows (or one larger pair), each with its
    // own prefix in pw0 at [bp[b] + b, bp[b + 1] + b]; and the scan tiles of the largest one
    const int64_t cap = h->corpus_pairs_batch > 0 ? h->corpus_pairs_batch : CORPUS_PAIRS_BATCH;
    std::vector<int64_t> bp{0};
    std::vector<long long> pw0;
    pw0.reserve((size_t)n_pairs + 1);
    int64_t max_bw = 0, max_tiles = 0;
    for (int64_t i = 0; i < n_pairs;) {
        int64_t j = i + 1;
        while (j < n_pairs && P[j + 1] - P[i] <= cap) ++j;
        for (int64_t q = i; q <= j; ++q) pw0.push_back(P[q] - P[i]);
        int64_t tiles = 0;
        for (int64_t a = i; a < j;) {                                 // runs of one model
            int64_t e = a + 1;
            while (e < j && pairs[e].x == pairs[a].x) ++e;
            tiles += (P[e] - P[a] + 63) / 64;
            a = e;
        }
        max_bw = std::max<int64_t>(max_bw, P[j] - P[i]);
        max_tiles = std::max(max_tiles, tiles);
        bp.push_back(j);
        i = j;
    }
    const int64_t n_batches = (int64_t)bp.size() - 1;
    const long long Wp = P[n_pairs];
    const bool own_raw = !d_raw && (reduce || hits) && Wp > 0;
    CorpusPoolSizes ps;
    ps.raw = own_raw ? (size_t)max_bw : 0;
    ps.pairs = (size_t)n_pairs;
    ps.pw0 = pw0.size();
    ps.starts = (size_t)max_bw;
    ps.tiles = (size_t)max_tiles;
    rc = corpus_reserve(h, plan, n_rec, ps, s);
    if (rc != PB_OK) return rc;
    auto launch = [&]() -> int {
        rc = corpus_k1(h, plan, d_pcm, n_rec, divisor, schedule, chunk, s);
        if (rc != PB_OK) return rc;
        if (hits) CK(cudaMemsetAsync(d_n_hits, 0, sizeof(unsigned long long), s));
        CK(cudaMemcpyAsync(h->d_pp_pairs.get(), pairs.data(), pairs.size() * sizeof(int2), cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(h->d_pp_pw0.get(), pw0.data(), pw0.size() * sizeof(long long), cudaMemcpyHostToDevice, s));
        ProfScope prof(h, 1, s);
        const K2In in = corpus_k2in(h);
        const uint4* slots = h->d_pool_slots.get();
        std::vector<PairTile> tiles;
        for (int64_t b = 0; b < n_batches; ++b) {
            const int64_t p0 = bp[b], p1 = bp[b + 1], nb = p1 - p0;
            const long long q0 = P[p0], nw = P[p1] - q0;
            const long long* bpw0 = h->d_pp_pw0.get() + p0 + b;
            const int2* bpairs = h->d_pp_pairs.get() + p0;
            float* raw = own_raw ? h->d_cp_raw.get() : d_raw ? d_raw + q0 : nullptr;
            double* conf = d_conf ? d_conf + q0 : nullptr;
            if (nw > 0) {
                pairs_windows_kernel<<<(unsigned)((nw + 255) / 256), 256, 0, s>>>(bpw0, bpairs, (int)nb, nw, h->d_cw_win0.get(),
                                                                                 h->d_cw_starts.get(), h->d_pp_starts.get());
                CK(cudaGetLastError());
                const int64_t n_keras = pair_tiles(h, pairs, P, p0, p1, tiles);
                CK(cudaMemcpyAsync(h->d_pp_tiles.get(), tiles.data(), tiles.size() * sizeof(PairTile), cudaMemcpyHostToDevice, s));
                PairsCorpus c{};
                c.slots = slots; c.starts = h->d_pp_starts.get(); c.raw = raw; c.conf = conf;
                c.tiles = h->d_pp_tiles.get(); c.n_tiles = n_keras;
                rc = launch_pairs_corpus<true>(c, in, s);
                if (rc != PB_OK) return rc;
                c.tiles += n_keras; c.n_tiles = (int64_t)tiles.size() - n_keras;
                rc = launch_pairs_corpus<false>(c, in, s);
                if (rc != PB_OK) return rc;
            }
            if (reduce) {
                // one "recording" per pair of the batch, one row
                CorpusTrig t = corpus_trig(h, nb, nw, schedule, chunk, threshold);
                t.win0 = bpw0;
                t.raw = raw; t.conf = conf;
                t.fired = d_fired ? d_fired + q0 : nullptr;
                t.activations = d_activations ? d_activations + p0 : nullptr;
                t.above = d_above ? d_above + p0 : nullptr;
                t.sum = d_sum ? d_sum + p0 : nullptr;
                CorpusPairsDP dp{slots, bpairs, trigger_reset(2 * chunk)};
                const unsigned per = CORPUS_TRIG_THREADS / 32;
                corpus_trigger_kernel<<<dim3((unsigned)((nb + per - 1) / per), 1), CORPUS_TRIG_THREADS, 0, s>>>(t, dp);
                CK(cudaGetLastError());
            }
            if (hits && nw > 0) {
                PairsHits H{};
                H.raw = raw; H.pw0 = bpw0; H.slots = slots; H.pairs = bpairs;
                H.n = nw; H.q_base = q0; H.capacity = hit_capacity; H.n_pairs = (int)nb;
                H.threshold = hit_threshold; H.hits = d_hits; H.n_hits = d_n_hits;
                pairs_hits_kernel<<<(unsigned)((nw + 255) / 256), 256, 0, s>>>(H);
                CK(cudaGetLastError());
            }
        }
        return PB_OK;
    };
    return corpus_done(h, s, launch());
}

// ------------------------------------------------------------------------------------------------
// pool models over labelled clips (dataset.cuh)

PB_API int pb_score_dataset(pb_handle* h, const int16_t* d_pcm, const int64_t* h_offsets, int64_t n_rec,
                            const uint8_t* h_targets, const int32_t* h_model_ids, int64_t k,
                            const int32_t* h_pair_rows, const int32_t* h_pair_recs, int64_t n_pairs,
                            int32_t divisor, int64_t max_samples, const double* h_thresholds, int32_t n_thr,
                            float* d_raw, int64_t* d_count, int64_t* d_hist, int64_t* d_fit,
                            double miss_threshold, int64_t* d_miss, int64_t miss_capacity, unsigned long long* d_n_miss,
                            void* stream) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    int rc = check_corpus(h, d_pcm, h_offsets, n_rec, divisor, PB_CORPUS_LISTENER, 1, d_raw, false, nullptr, nullptr);
    if (rc != PB_OK) return rc;
    const bool misses = d_n_miss != nullptr, stats = d_count || d_hist || d_fit || misses;
    if (!d_raw && !stats) return fail(PB_ERR_INVALID, "every output is null");
    if (!h->pool) return fail(PB_ERR_STATE, "no model pool: call pb_set_pool first");
    if (max_samples < 1) return fail(PB_ERR_INVALID, "max_samples = %lld must be >= 1", (long long)max_samples);
    if (n_rec > 0 && !h_targets) return fail(PB_ERR_INVALID, "null h_targets");
    for (int64_t r = 0; r < n_rec; ++r)
        if (h_offsets[r + 1] == h_offsets[r]) return fail(PB_ERR_INVALID, "recording %lld is empty: cannot vectorize empty audio", (long long)r);
    if (k < 0 || k > INT32_MAX / 2) return fail(PB_ERR_INVALID, "k = %lld outside [0, 2^30)", (long long)k);
    if (k > 0 && !h_model_ids) return fail(PB_ERR_INVALID, "null h_model_ids");
    for (int64_t i = 0; i < k; ++i) {
        const int32_t m = h_model_ids[i];
        if (m < 0 || m >= h->pool_models)
            return fail(PB_ERR_INVALID, "model id %d (entry %lld) outside [0, max_models = %d)", m, (long long)i, h->pool_models);
        if (h->pool_cd_of[m] == h->pool_cd.end())
            return fail(PB_ERR_INVALID, "pool slot %d (entry %lld) holds no model: pb_pool_load it first", m, (long long)i);
    }
    if (n_pairs < 0 || n_pairs > INT32_MAX) return fail(PB_ERR_INVALID, "n_pairs = %lld outside [0, 2^31)", (long long)n_pairs);
    const bool by_pairs = n_pairs > 0;
    if (by_pairs && (!h_pair_rows || !h_pair_recs)) return fail(PB_ERR_INVALID, "null h_pair_rows or h_pair_recs");
    for (int64_t i = 0; i < n_pairs; ++i) {
        const int32_t row = h_pair_rows[i], r = h_pair_recs[i];
        if (row < 0 || row >= k) return fail(PB_ERR_INVALID, "row %d (pair %lld) outside [0, k = %lld)", row, (long long)i, (long long)k);
        if (r < 0 || r >= n_rec)
            return fail(PB_ERR_INVALID, "recording id %d (pair %lld) outside [0, n_rec = %lld)", r, (long long)i, (long long)n_rec);
    }
    if (n_thr < 0 || n_thr > DS_MAX_THR) return fail(PB_ERR_INVALID, "n_thr = %d outside [0, %d]", n_thr, DS_MAX_THR);
    if (d_hist && n_thr < 1) return fail(PB_ERR_INVALID, "d_hist needs at least one threshold");
    if (n_thr > 0 && !h_thresholds) return fail(PB_ERR_INVALID, "null h_thresholds");
    std::vector<float> thr((size_t)n_thr);
    for (int i = 0; i < n_thr; ++i) {
        thr[i] = (float)h_thresholds[i];
        if (!(i == 0 ? thr[i] == thr[i] : thr[i] > thr[i - 1]))
            return fail(PB_ERR_INVALID, "threshold %d = %g: rounded to float32, thresholds must be strictly ascending", i, h_thresholds[i]);
    }
    if (miss_capacity < 0) return fail(PB_ERR_INVALID, "miss_capacity = %lld is negative", (long long)miss_capacity);
    if (miss_capacity > 0 && !d_miss) return fail(PB_ERR_INVALID, "null d_miss with miss_capacity = %lld", (long long)miss_capacity);
    if (d_miss && !misses) return fail(PB_ERR_INVALID, "d_miss without d_n_miss");
    if (d_fit) {
        // the fit's int64 sums hold 2^24 entries of one (row, label)
        const int64_t limit = 1ll << 24;
        if (by_pairs) {
            std::vector<int64_t> per((size_t)k * 2, 0);
            for (int64_t i = 0; i < n_pairs; ++i)
                if (++per[(size_t)h_pair_rows[i] * 2 + (h_targets[h_pair_recs[i]] != 0)] > limit)
                    return fail(PB_ERR_INVALID, "row %d has more than 2^24 entries of one label: split the call", h_pair_rows[i]);
        } else {
            int64_t pos = 0;
            for (int64_t r = 0; r < n_rec; ++r) pos += h_targets[r] != 0;
            if (k > 0 && std::max(pos, n_rec - pos) > limit)
                return fail(PB_ERR_INVALID, "%lld recordings of one label, more than 2^24: split the call", (long long)std::max(pos, n_rec - pos));
        }
    }
    CK(cudaSetDevice(h->cfg.device));
    cudaStream_t s = (cudaStream_t)stream;
    const int bins = 2 * n_thr + 1;
    auto zero = [&]() -> int {
        if (d_count) CK(cudaMemsetAsync(d_count, 0, (size_t)k * 2 * sizeof(int64_t), s));
        if (d_hist) CK(cudaMemsetAsync(d_hist, 0, (size_t)k * 2 * bins * sizeof(int64_t), s));
        if (d_fit) CK(cudaMemsetAsync(d_fit, 0, (size_t)k * 6 * sizeof(int64_t), s));
        if (misses) CK(cudaMemsetAsync(d_n_miss, 0, sizeof(unsigned long long), s));
        return PB_OK;
    };
    if (n_rec == 0 || k == 0) return zero();
    const CorpusPlan plan = corpus_plan(h, d_pcm, h_offsets, n_rec, PB_CORPUS_LISTENER, 1, max_samples);
    // entries per batch: all of them into the caller's d_raw, else as many as the capped raw buffer holds; the cross product
    // in whole rows, pairs in runs of consecutive pairs
    const int NM = h->corpus_pool_nm ? h->corpus_pool_nm : CORPUS_POOL_NM;
    int64_t rows = k, cap = 0;
    std::vector<int2> groups, slot_pairs, row_pairs;
    std::vector<int64_t> g0;
    std::vector<long long> P;
    CorpusPoolSizes ps;
    ps.thr = d_hist ? (size_t)n_thr : 0;
    ps.targets = stats ? (size_t)n_rec : 0;
    if (by_pairs) {
        cap = std::min<int64_t>(n_pairs, h->corpus_pairs_batch > 0 ? h->corpus_pairs_batch : CORPUS_PAIRS_BATCH);
        slot_pairs.resize((size_t)n_pairs);
        row_pairs.resize((size_t)n_pairs);
        P.resize((size_t)n_pairs + 1);
        for (int64_t i = 0; i < n_pairs; ++i) {
            slot_pairs[i] = make_int2(h_model_ids[h_pair_rows[i]], h_pair_recs[i]);
            row_pairs[i] = make_int2(h_pair_rows[i], h_pair_recs[i]);
            P[i] = i;
        }
        P[n_pairs] = n_pairs;
        ps.raw = !d_raw ? (size_t)cap : 0;
        ps.pairs = (size_t)n_pairs;
        ps.pw0 = (size_t)cap + 1;
        ps.starts = (size_t)cap;
        for (int64_t p0 = 0; p0 < n_pairs; p0 += cap) {               // the scan tiles of the largest batch
            const int64_t p1 = std::min(n_pairs, p0 + cap);
            size_t tiles = 0;
            for (int64_t a = p0, e; a < p1; a = e) {
                for (e = a + 1; e < p1 && slot_pairs[e].x == slot_pairs[a].x;) ++e;
                tiles += (size_t)((e - a + 63) / 64);
            }
            ps.tiles = std::max(ps.tiles, tiles);
        }
    } else {
        if (!d_raw) {
            rows = std::max<int64_t>(1, CORPUS_POOL_RAW_CAP / (4 * n_rec));
            if (h->corpus_pool_rows > 0) rows = std::min<int64_t>(rows, h->corpus_pool_rows);
            rows = std::min<int64_t>(rows, k);
        }
        pool_corpus_groups(h, h_model_ids, k, rows, NM, groups, g0);
        ps.groups = groups.size();
        ps.raw = !d_raw ? (size_t)(rows * n_rec) : 0;
    }
    rc = corpus_reserve(h, plan, n_rec, ps, s);
    if (rc != PB_OK) return rc;
    auto launch = [&]() -> int {
        rc = corpus_k1(h, plan, d_pcm, n_rec, divisor, PB_CORPUS_LISTENER, 1, s);
        if (rc != PB_OK) return rc;
        rc = zero();
        if (rc != PB_OK) return rc;
        if (d_hist) CK(cudaMemcpyAsync(h->d_ds_thr.get(), thr.data(), thr.size() * sizeof(float), cudaMemcpyHostToDevice, s));
        if (stats) CK(cudaMemcpyAsync(h->d_ds_targets.get(), h_targets, (size_t)n_rec, cudaMemcpyHostToDevice, s));
        ProfScope prof(h, 1, s);
        const K2In in = corpus_k2in(h);
        DatasetStats D{};
        D.targets = h->d_ds_targets.get(); D.thr = d_hist ? h->d_ds_thr.get() : nullptr; D.n_thr = n_thr;
        D.count = d_count; D.hist = d_hist; D.fit = d_fit;
        D.miss_thr = (float)miss_threshold; D.miss = d_miss; D.capacity = miss_capacity; D.n_miss = d_n_miss;
        if (!by_pairs) {
            CK(cudaMemcpyAsync(h->d_cp_groups.get(), groups.data(), groups.size() * sizeof(int2), cudaMemcpyHostToDevice, s));
            const bool split = pool_corpus_keras(NM);
            const int order = h->corpus_pool_order >= 0 ? h->corpus_pool_order : CORPUS_POOL_GROUPS_FAST;
            for (int64_t b0 = 0, b = 0; b0 < k; b0 += rows, ++b) {
                const int64_t nb = std::min<int64_t>(k, b0 + rows) - b0;
                float* raw = d_raw ? d_raw + b0 * n_rec : h->d_cp_raw.get();
                PoolCorpus c{};
                c.slots = h->d_pool_slots.get(); c.n_tiles = (n_rec + 63) / 64; c.raw = raw; c.W = n_rec; c.groups_fast = order;
                for (int ka = 0; ka < 2; ++ka) {
                    c.groups = h->d_cp_groups.get() + g0[2 * b + ka] * NM;
                    c.n_groups = g0[2 * b + ka + 1] - g0[2 * b + ka];
                    rc = launch_pool_corpus_nm(NM, split && ka == 1, c, in, s);
                    if (rc != PB_OK) return rc;
                }
                if (!stats) continue;
                const unsigned gx = (unsigned)((n_rec + DS_THREADS * DS_ITERS - 1) / (DS_THREADS * DS_ITERS));
                for (int64_t y0 = 0; y0 < nb; y0 += 65535) {          // gridDim.y
                    D.raw = raw + y0 * n_rec; D.row0 = (int)(b0 + y0); D.n = n_rec;
                    dataset_stats_kernel<false><<<dim3(gx, (unsigned)std::min<int64_t>(65535, nb - y0)), DS_THREADS, 0, s>>>(D);
                    CK(cudaGetLastError());
                }
            }
            return PB_OK;
        }
        CK(cudaMemcpyAsync(h->d_pp_pairs.get(), row_pairs.data(), row_pairs.size() * sizeof(int2), cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(h->d_pp_pw0.get(), P.data(), (size_t)(cap + 1) * sizeof(long long), cudaMemcpyHostToDevice, s));
        std::vector<PairTile> tiles;
        for (int64_t p0 = 0; p0 < n_pairs; p0 += cap) {
            const int64_t p1 = std::min(n_pairs, p0 + cap), nb = p1 - p0;
            const int2* bpairs = h->d_pp_pairs.get() + p0;
            float* raw = d_raw ? d_raw + p0 : h->d_cp_raw.get();
            // one pair-window per pair: the batch's prefix is 0 .. nb
            pairs_windows_kernel<<<(unsigned)((nb + 255) / 256), 256, 0, s>>>(h->d_pp_pw0.get(), bpairs, (int)nb, nb, h->d_cw_win0.get(),
                                                                             h->d_cw_starts.get(), h->d_pp_starts.get());
            CK(cudaGetLastError());
            const int64_t n_keras = pair_tiles(h, slot_pairs, P, p0, p1, tiles);
            CK(cudaMemcpyAsync(h->d_pp_tiles.get(), tiles.data(), tiles.size() * sizeof(PairTile), cudaMemcpyHostToDevice, s));
            PairsCorpus c{};
            c.slots = h->d_pool_slots.get(); c.starts = h->d_pp_starts.get(); c.raw = raw;
            c.tiles = h->d_pp_tiles.get(); c.n_tiles = n_keras;
            rc = launch_pairs_corpus<true>(c, in, s);
            if (rc != PB_OK) return rc;
            c.tiles += n_keras; c.n_tiles = (int64_t)tiles.size() - n_keras;
            rc = launch_pairs_corpus<false>(c, in, s);
            if (rc != PB_OK) return rc;
            if (!stats) continue;
            D.raw = raw; D.pairs = bpairs; D.n = nb; D.base = p0;
            dataset_stats_kernel<true><<<(unsigned)((nb + DS_THREADS - 1) / DS_THREADS), DS_THREADS, 0, s>>>(D);
            CK(cudaGetLastError());
        }
        return PB_OK;
    };
    return corpus_done(h, s, launch());
}

// ------------------------------------------------------------------------------------------------
// training (train.cuh)

constexpr size_t TRAIN_WS_CAP = size_t(256) << 20;     // workspace of one group of rows
constexpr size_t TRAIN_ALIGN = 256;

// The fused family's front end, which pb_vectorize_clips and the training kernels cover.
static int check_train_front_end(const pb_handle* h) {
    if (h->cfg.use_delta || h->feat > TR_MAX_F)
        return fail(PB_ERR_UNSUPPORTED, "training covers the fused family's front end (feature size <= %d, no deltas); this handle "
                    "has feature size %d%s", TR_MAX_F, h->feat, h->cfg.use_delta ? " with deltas" : "");
    if (train_smem(h->cfg.n_features) > 227 * 1024)
        return fail(PB_ERR_UNSUPPORTED, "n_features = %d: the training kernel keeps at most 112 steps in shared memory", h->cfg.n_features);
    return PB_OK;
}

PB_API int pb_vectorize_clips(pb_handle* h, const int16_t* d_pcm, const int64_t* h_offsets, int64_t n_rec, int32_t divisor,
                              int64_t max_samples, float* d_inputs, void* stream) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    int rc = check_train_front_end(h);
    if (rc != PB_OK) return rc;
    rc = check_corpus(h, d_pcm, h_offsets, n_rec, divisor, PB_CORPUS_LISTENER, 1, d_inputs, true, nullptr, nullptr);
    if (rc != PB_OK) return rc;
    if (max_samples < 1) return fail(PB_ERR_INVALID, "max_samples = %lld must be >= 1", (long long)max_samples);
    for (int64_t r = 0; r < n_rec; ++r)
        if (h_offsets[r + 1] == h_offsets[r]) return fail(PB_ERR_INVALID, "recording %lld is empty: cannot vectorize empty audio", (long long)r);
    if (n_rec == 0) return PB_OK;
    CK(cudaSetDevice(h->cfg.device));
    cudaStream_t s = (cudaStream_t)stream;
    const CorpusPlan plan = corpus_plan(h, d_pcm, h_offsets, n_rec, PB_CORPUS_LISTENER, 1, max_samples);
    rc = corpus_reserve(h, plan, n_rec, CorpusPoolSizes{}, s);
    if (rc != PB_OK) return rc;
    auto launch = [&]() -> int {
        rc = corpus_k1(h, plan, d_pcm, n_rec, divisor, PB_CORPUS_LISTENER, 1, s);
        if (rc != PB_OK) return rc;
        const int T = h->cfg.n_features, F = h->feat;
        const long long total = (long long)n_rec * T * F;
        vectorize_gather_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(h->d_cw_rows.get(), h->d_cw_starts.get(), h->row_stride,
                                                                               T, F, n_rec, d_inputs);
        CK(cudaGetLastError());
        return PB_OK;
    };
    return corpus_done(h, s, launch());
}

PB_API int pb_train_opts_default(pb_train_opts* o) {
    if (!o) return fail(PB_ERR_INVALID, "opts is null");
    o->epochs = 10; o->epoch0 = 0; o->batch_size = 5000;
    o->lr = 0.001f; o->rho = 0.9f; o->epsilon = 1e-7f;
    o->loss_bias = 0.8f; o->dropout = 0.2f;
    return PB_OK;
}

// The entries of a training call: row r's entry j uses clip ent[off[r] + j].
struct TrainEntries {
    std::vector<int64_t> off;        // [k + 1]
    std::vector<int> ent;
};

// A group of consecutive rows with entries, trained together, and its tile tables: batch b's gradient tiles are
// tiles[tile0[b] .. tile0[b + 1]), its row updates steps[step0[b] .. step0[b + 1]).
struct TrainGroup {
    std::vector<int> rows;
    int64_t e0 = 0, n = 0;           // entries [e0, e0 + n) of TrainEntries::ent
    std::vector<int> seg;            // [rows + 1] group-local entry offsets
    std::vector<TrainTile> tiles;
    std::vector<TrainStep> steps;
    std::vector<int64_t> tile0, step0;
    int64_t max_tiles = 0;
    size_t sort_bytes = 0;
};

// Checks the arguments both training calls share and lists the entries.
static int check_train(const pb_handle* h, const float* d_inputs, int64_t n_rec, const uint8_t* h_targets, const pb_train_row* h_rows,
                       int64_t k, const int32_t* h_pair_rows, const int32_t* h_pair_recs, int64_t n_pairs, TrainEntries& te) {
    int rc = check_train_front_end(h);
    if (rc != PB_OK) return rc;
    if (k < 0 || k > INT32_MAX / 2) return fail(PB_ERR_INVALID, "k = %lld outside [0, 2^30)", (long long)k);
    if (k > 0 && !h_rows) return fail(PB_ERR_INVALID, "null h_rows");
    for (int64_t i = 0; i < k; ++i) {
        const pb_train_row& r = h_rows[i];
        if (r.hidden < 1 || r.hidden > TR_MAX_H) return fail(PB_ERR_INVALID, "row %lld: hidden = %d outside [1, %d]", (long long)i, r.hidden, TR_MAX_H);
        if ((r.activation != PB_ACT_LINEAR && r.activation != PB_ACT_TANH) ||
            (r.recurrent_activation != PB_RACT_HARD_SIGMOID && r.recurrent_activation != PB_RACT_SIGMOID))
            return fail(PB_ERR_INVALID, "row %lld: unknown activation codes (%d, %d)", (long long)i, r.activation, r.recurrent_activation);
    }
    if (n_rec < 0 || n_rec > INT32_MAX) return fail(PB_ERR_INVALID, "n_rec = %lld outside [0, 2^31)", (long long)n_rec);
    if (n_pairs < 0 || n_pairs > INT32_MAX) return fail(PB_ERR_INVALID, "n_pairs = %lld outside [0, 2^31)", (long long)n_pairs);
    const bool by_pairs = n_pairs > 0;
    if (by_pairs && (!h_pair_rows || !h_pair_recs)) return fail(PB_ERR_INVALID, "null h_pair_rows or h_pair_recs");
    for (int64_t i = 0; i < n_pairs; ++i) {
        const int32_t row = h_pair_rows[i], r = h_pair_recs[i];
        if (row < 0 || row >= k) return fail(PB_ERR_INVALID, "row %d (pair %lld) outside [0, k = %lld)", row, (long long)i, (long long)k);
        if (r < 0 || r >= n_rec)
            return fail(PB_ERR_INVALID, "clip %d (pair %lld) outside [0, n_rec = %lld)", r, (long long)i, (long long)n_rec);
    }
    const int64_t total = by_pairs ? n_pairs : k * n_rec;
    if (total > 0 && (!d_inputs || !h_targets)) return fail(PB_ERR_INVALID, "null d_inputs or h_targets");
    // one row's entries must fit one group's workspace
    const int64_t per_row_max = (int64_t)(TRAIN_WS_CAP / 64);
    te.off.assign((size_t)k + 1, 0);
    if (by_pairs) {
        for (int64_t i = 0; i < n_pairs; ++i) ++te.off[(size_t)h_pair_rows[i] + 1];
    } else {
        for (int64_t i = 0; i < k; ++i) te.off[(size_t)i + 1] = n_rec;
    }
    for (int64_t i = 0; i < k; ++i) {
        if (te.off[(size_t)i + 1] > per_row_max)
            return fail(PB_ERR_INVALID, "row %lld has %lld entries, more than %lld: split the call", (long long)i,
                        (long long)te.off[(size_t)i + 1], (long long)per_row_max);
        te.off[(size_t)i + 1] += te.off[(size_t)i];
    }
    te.ent.resize((size_t)total);
    if (by_pairs) {
        std::vector<int64_t> at(te.off.begin(), te.off.end() - 1);
        for (int64_t i = 0; i < n_pairs; ++i) te.ent[(size_t)at[(size_t)h_pair_rows[i]]++] = h_pair_recs[i];
    } else {
        for (int64_t i = 0; i < k; ++i)
            for (int64_t r = 0; r < n_rec; ++r) te.ent[(size_t)(i * n_rec + r)] = (int)r;
    }
    return PB_OK;
}

// Entries per batch of row with n entries at batch size bs: tiles of TR_TILE entries.
static int64_t train_tiles(int64_t n, int64_t bs) {
    int64_t t = 0;
    for (int64_t b0 = 0; b0 < n; b0 += bs) t += (std::min(bs, n - b0) + TR_TILE - 1) / TR_TILE;
    return t;
}

// Groups of consecutive rows with entries whose workspace stays under TRAIN_WS_CAP, with their tile tables.
static std::vector<TrainGroup> train_groups(const TrainEntries& te, int64_t k, int64_t bs) {
    std::vector<TrainGroup> out;
    size_t bytes = 0;
    for (int64_t r = 0; r < k; ++r) {
        const int64_t n = te.off[(size_t)r + 1] - te.off[(size_t)r];
        if (n == 0) continue;
        const int64_t b = std::min(bs, n), nb = (n + bs - 1) / bs;
        const size_t cost = (size_t)n * 40 + (size_t)((b + TR_TILE - 1) / TR_TILE) * (TR_STRIDE * 4 + 8) +
                            (size_t)train_tiles(n, bs) * sizeof(TrainTile) + (size_t)nb * sizeof(TrainStep) + 64;
        if (out.empty() || bytes + cost > TRAIN_WS_CAP || out.back().rows.size() >= 65535) {
            out.emplace_back();
            out.back().e0 = te.off[(size_t)r];
            out.back().seg.push_back(0);
            bytes = 0;
        }
        TrainGroup& g = out.back();
        g.rows.push_back((int)r);
        g.n += n;
        g.seg.push_back((int)g.n);
        bytes += cost;
    }
    for (TrainGroup& g : out) {
        int64_t nb_max = 0;
        for (size_t i = 0; i < g.rows.size(); ++i) nb_max = std::max<int64_t>(nb_max, (g.seg[i + 1] - g.seg[i] + bs - 1) / bs);
        for (int64_t b = 0; b < nb_max; ++b) {
            g.tile0.push_back((int64_t)g.tiles.size());
            g.step0.push_back((int64_t)g.steps.size());
            int t_launch = 0;
            for (size_t i = 0; i < g.rows.size(); ++i) {
                const int64_t n = g.seg[i + 1] - g.seg[i], b0 = b * bs;
                if (b0 >= n) continue;
                const int B = (int)std::min(bs, n - b0);
                const int t0 = t_launch;
                for (int q = 0; q < B; q += TR_TILE)
                    g.tiles.push_back(TrainTile{g.rows[i], g.seg[i], (int)b0 + q, std::min(TR_TILE, B - q), B}), ++t_launch;
                g.steps.push_back(TrainStep{g.rows[i], t0, t_launch, b0 + bs >= n ? TR_LAST : 0, (int)n});
            }
            g.max_tiles = std::max<int64_t>(g.max_tiles, t_launch);
        }
        g.tile0.push_back((int64_t)g.tiles.size());
        g.step0.push_back((int64_t)g.steps.size());
    }
    return out;
}

// Carves typed arrays out of the training arena (a null base only measures).
struct TrainCarve {
    uint8_t* base;
    size_t at = 0;
    template <typename T> T* take(size_t n) {
        at = (at + TRAIN_ALIGN - 1) / TRAIN_ALIGN * TRAIN_ALIGN;
        T* p = base ? reinterpret_cast<T*>(base + at) : nullptr;
        at += std::max<size_t>(n, 1) * sizeof(T);
        return p;
    }
};

struct TrainWs {
    TrainRowDev* rows; uint8_t* targets; double* loss_acc;
    int* ent; int* order; int* vals; uint64_t* keys; uint64_t* keys2; int* seg; int* seg_row;
    TrainTile* tiles; TrainStep* steps; float* part; double* part_loss; void* sort_tmp;
};

static TrainWs train_layout(uint8_t* base, int64_t k, int64_t n_rec, int64_t n, int64_t rows, int64_t tiles, int64_t steps,
                            int64_t max_tiles, size_t sort_bytes, size_t* bytes) {
    TrainCarve c{base};
    TrainWs w{};
    w.rows = c.take<TrainRowDev>((size_t)k); w.targets = c.take<uint8_t>((size_t)n_rec); w.loss_acc = c.take<double>((size_t)k);
    w.ent = c.take<int>((size_t)n); w.order = c.take<int>((size_t)n); w.vals = c.take<int>((size_t)n);
    w.keys = c.take<uint64_t>((size_t)n); w.keys2 = c.take<uint64_t>((size_t)n);
    w.seg = c.take<int>((size_t)rows + 1); w.seg_row = c.take<int>((size_t)rows);
    w.tiles = c.take<TrainTile>((size_t)tiles); w.steps = c.take<TrainStep>((size_t)steps);
    w.part = c.take<float>((size_t)max_tiles * TR_STRIDE); w.part_loss = c.take<double>((size_t)max_tiles);
    w.sort_tmp = c.take<uint8_t>(sort_bytes);
    if (bytes) *bytes = c.at;
    return w;
}

// Shared body of pb_train (train = true: shuffle, batches, RMSprop) and pb_train_loss (one batch per row in request order,
// the gradient to d_grad).
static int train_run(pb_handle* h, const float* d_inputs, int64_t n_rec, const uint8_t* h_targets, const pb_train_row* h_rows,
                     int64_t k, const TrainEntries& te, bool train, int epochs, int epoch0, int64_t bs, float lr, float rho,
                     float eps, float loss_bias, float dropout, const float* d_weights_in, float* d_weights, float* d_rms,
                     double* d_loss, float* d_grad, cudaStream_t s) {
    CK(cudaSetDevice(h->cfg.device));
    std::vector<TrainGroup> groups = train_groups(te, k, train ? bs : std::numeric_limits<int64_t>::max() / 2);
    int64_t rows_max = 0, n_max = 0, tiles_max = 0, steps_max = 0, ptiles_max = 0;
    size_t sort_max = 0;
    for (TrainGroup& g : groups) {
        if (train) {
            size_t sb = 0;
            CK(cub::DeviceSegmentedSort::StableSortPairs(nullptr, sb, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int*)nullptr,
                                                         (int*)nullptr, (int)g.n, (int)g.rows.size(), (const int*)nullptr,
                                                         (const int*)nullptr, s));
            g.sort_bytes = sb;
        }
        rows_max = std::max<int64_t>(rows_max, (int64_t)g.rows.size());
        n_max = std::max(n_max, g.n);
        tiles_max = std::max<int64_t>(tiles_max, (int64_t)g.tiles.size());
        steps_max = std::max<int64_t>(steps_max, (int64_t)g.steps.size());
        ptiles_max = std::max(ptiles_max, g.max_tiles);
        sort_max = std::max(sort_max, g.sort_bytes);
    }
    size_t bytes = 0;
    train_layout(nullptr, k, n_rec, n_max, rows_max, tiles_max, steps_max, ptiles_max, sort_max, &bytes);
    if (!h->corpus_ev) CK(cudaEventCreateWithFlags(&h->corpus_ev, cudaEventDisableTiming));
    if (h->d_tr_ws.size() < bytes) {
        DevArray<uint8_t> fresh;
        const cudaError_t e = fresh.alloc(bytes);
        if (e != cudaSuccess) {
            cudaGetLastError();
            return fail(PB_ERR_CUDA, "training workspace allocation failed (%zu bytes): %s", bytes, cudaGetErrorString(e));
        }
        CK(cudaEventSynchronize(h->corpus_ev));                     // the previous call may still use the arena
        h->d_tr_ws = std::move(fresh);
    }
    CK(ensure_dyn_smem(train_grad_kernel, train_smem(h->cfg.n_features)));
    CK(cudaStreamWaitEvent(s, h->corpus_ev, 0));
    const TrainWs w = train_layout(h->d_tr_ws.get(), k, n_rec, n_max, rows_max, tiles_max, steps_max, ptiles_max, sort_max, nullptr);
    auto launch = [&]() -> int {
        const int n_loss = train ? epochs : 1;
        if (d_loss) {
            const std::vector<double> nan((size_t)k * n_loss, std::numeric_limits<double>::quiet_NaN());
            CK(cudaMemcpyAsync(d_loss, nan.data(), nan.size() * sizeof(double), cudaMemcpyHostToDevice, s));
        }
        if (groups.empty()) return PB_OK;
        std::vector<TrainRowDev> rd((size_t)k);
        for (int64_t i = 0; i < k; ++i)
            rd[i] = TrainRowDev{h_rows[i].hidden, h_rows[i].activation, h_rows[i].recurrent_activation, h_rows[i].seed};
        CK(cudaMemcpyAsync(w.rows, rd.data(), rd.size() * sizeof(TrainRowDev), cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(w.targets, h_targets, (size_t)n_rec, cudaMemcpyHostToDevice, s));
        CK(cudaMemsetAsync(w.loss_acc, 0, (size_t)k * sizeof(double), s));
        ProfScope prof(h, 1, s);
        const float scale = 1.0f / (1.0f - dropout);
        for (const TrainGroup& g : groups) {
            CK(cudaMemcpyAsync(w.ent, te.ent.data() + g.e0, (size_t)g.n * sizeof(int), cudaMemcpyHostToDevice, s));
            CK(cudaMemcpyAsync(w.seg, g.seg.data(), g.seg.size() * sizeof(int), cudaMemcpyHostToDevice, s));
            CK(cudaMemcpyAsync(w.seg_row, g.rows.data(), g.rows.size() * sizeof(int), cudaMemcpyHostToDevice, s));
            CK(cudaMemcpyAsync(w.tiles, g.tiles.data(), g.tiles.size() * sizeof(TrainTile), cudaMemcpyHostToDevice, s));
            CK(cudaMemcpyAsync(w.steps, g.steps.data(), g.steps.size() * sizeof(TrainStep), cudaMemcpyHostToDevice, s));
            int64_t seg_max = 0;
            for (size_t i = 0; i < g.rows.size(); ++i) seg_max = std::max<int64_t>(seg_max, g.seg[i + 1] - g.seg[i]);
            for (int ep = 0; ep < (train ? epochs : 1); ++ep) {
                const long long epoch = (long long)epoch0 + ep;
                if (train) {
                    const dim3 grid((unsigned)std::min<int64_t>((seg_max + 255) / 256, 64), (unsigned)g.rows.size());
                    train_keys_kernel<<<grid, 256, 0, s>>>(w.rows, w.seg, w.seg_row, (int)g.rows.size(), epoch, w.keys, w.vals);
                    CK(cudaGetLastError());
                    size_t sb = g.sort_bytes;
                    CK(cub::DeviceSegmentedSort::StableSortPairs(w.sort_tmp, sb, w.keys, w.keys2, w.vals, w.order, (int)g.n,
                                                                 (int)g.rows.size(), w.seg, w.seg + 1, s));
                }
                for (size_t b = 0; b + 1 < g.tile0.size(); ++b) {
                    TrainGrad G{};
                    G.weights = train ? d_weights : d_weights_in; G.rows = w.rows; G.inputs = d_inputs; G.targets = w.targets;
                    G.ent = w.ent; G.order = train ? w.order : nullptr; G.tiles = w.tiles + g.tile0[b];
                    G.part = w.part; G.part_loss = w.part_loss;
                    G.T = h->cfg.n_features; G.F = h->feat; G.epoch = epoch;
                    G.rate = dropout; G.scale = scale; G.loss_bias = loss_bias;
                    const unsigned nt = (unsigned)(g.tile0[b + 1] - g.tile0[b]);
                    train_grad_kernel<<<nt, TR_THREADS, train_smem(G.T), s>>>(G);
                    CK(cudaGetLastError());
                    TrainUpdate P{};
                    P.steps = w.steps + g.step0[b]; P.rows = w.rows; P.part = w.part; P.part_loss = w.part_loss;
                    P.weights = train ? d_weights : nullptr; P.rms = d_rms; P.grad = train ? nullptr : d_grad;
                    P.loss_acc = w.loss_acc; P.loss = d_loss; P.n_loss = n_loss; P.loss_col = ep; P.F = h->feat;
                    P.lr = lr; P.rho = rho; P.eps = eps;
                    train_update_kernel<<<(unsigned)(g.step0[b + 1] - g.step0[b]), TR_UPDATE_THREADS, 0, s>>>(P);
                    CK(cudaGetLastError());
                }
            }
        }
        return PB_OK;
    };
    return corpus_done(h, s, launch());
}

PB_API int pb_train(pb_handle* h, const float* d_inputs, int64_t n_rec, const uint8_t* h_targets, const pb_train_row* h_rows, int64_t k,
                    const int32_t* h_pair_rows, const int32_t* h_pair_recs, int64_t n_pairs, const pb_train_opts* opts,
                    float* d_weights, float* d_rms, double* d_loss, void* stream) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    if (!opts) return fail(PB_ERR_INVALID, "null opts");
    const pb_train_opts o = *opts;
    if (o.epochs < 1) return fail(PB_ERR_INVALID, "epochs = %d must be >= 1", o.epochs);
    if (o.epoch0 < 0) return fail(PB_ERR_INVALID, "epoch0 = %d is negative", o.epoch0);
    if (o.batch_size < 1) return fail(PB_ERR_INVALID, "batch_size = %d must be >= 1", o.batch_size);
    if (!(std::isfinite(o.lr) && o.lr >= 0.f)) return fail(PB_ERR_INVALID, "lr = %g must be finite and >= 0", o.lr);
    if (!(o.rho >= 0.f && o.rho < 1.f)) return fail(PB_ERR_INVALID, "rho = %g outside [0, 1)", o.rho);
    if (!(std::isfinite(o.epsilon) && o.epsilon >= 0.f)) return fail(PB_ERR_INVALID, "epsilon = %g must be finite and >= 0", o.epsilon);
    if (!(o.loss_bias >= 0.f && o.loss_bias <= 1.f)) return fail(PB_ERR_INVALID, "loss_bias = %g outside [0, 1]", o.loss_bias);
    if (!(o.dropout >= 0.f && o.dropout < 1.f)) return fail(PB_ERR_INVALID, "dropout = %g outside [0, 1)", o.dropout);
    TrainEntries te;
    const int rc = check_train(h, d_inputs, n_rec, h_targets, h_rows, k, h_pair_rows, h_pair_recs, n_pairs, te);
    if (rc != PB_OK) return rc;
    if (k > 0 && (!d_weights || !d_rms)) return fail(PB_ERR_INVALID, "null d_weights or d_rms");
    if (k == 0) return PB_OK;
    return train_run(h, d_inputs, n_rec, h_targets, h_rows, k, te, true, o.epochs, o.epoch0, o.batch_size, o.lr, o.rho, o.epsilon,
                     o.loss_bias, o.dropout, nullptr, d_weights, d_rms, d_loss, nullptr, (cudaStream_t)stream);
}

PB_API int pb_train_loss(pb_handle* h, const float* d_inputs, int64_t n_rec, const uint8_t* h_targets, const pb_train_row* h_rows,
                         int64_t k, const int32_t* h_pair_rows, const int32_t* h_pair_recs, int64_t n_pairs, float loss_bias,
                         float dropout, int32_t epoch, const float* d_weights, double* d_loss, float* d_grad, void* stream) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    if (!(loss_bias >= 0.f && loss_bias <= 1.f)) return fail(PB_ERR_INVALID, "loss_bias = %g outside [0, 1]", loss_bias);
    if (!(dropout >= 0.f && dropout < 1.f)) return fail(PB_ERR_INVALID, "dropout = %g outside [0, 1)", dropout);
    if (epoch < 0) return fail(PB_ERR_INVALID, "epoch = %d is negative", epoch);
    TrainEntries te;
    const int rc = check_train(h, d_inputs, n_rec, h_targets, h_rows, k, h_pair_rows, h_pair_recs, n_pairs, te);
    if (rc != PB_OK) return rc;
    if (k > 0 && !d_weights) return fail(PB_ERR_INVALID, "null d_weights");
    if (!d_loss && !d_grad) return fail(PB_ERR_INVALID, "d_loss and d_grad are both null");
    if (k == 0) return PB_OK;
    return train_run(h, d_inputs, n_rec, h_targets, h_rows, k, te, false, 1, epoch, 0, 0.f, 0.f, 0.f, loss_bias, dropout, d_weights,
                     nullptr, nullptr, d_loss, d_grad, (cudaStream_t)stream);
}

__global__ void read_window_kernel(K2In in, const int* ids, long long n, float* out) {
    // one thread per (item, row, column)
    const int Fb = in.F_base;
    long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    long long total = n * in.T * Fb;
    if (e >= total) return;
    int f = (int)(e % Fb);
    long long q = e / Fb;
    int t = (int)(q % in.T);
    long long i = q / in.T;
    int sid = ids ? ids[i] : (int)i;
    long long ns = in.n_samples[sid];
    long long rel = ns >= in.window ? (ns - in.window) / in.hop + 1 : 0;
    const float* row = ring_row(in, sid, rel, t);
    out[e] = row ? row[f] : 0.f;
}

PB_API int pb_read_window(pb_handle* h, const int32_t* d_ids, int64_t n, float* d_out, void* stream) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    if (n < 0 || n > h->cfg.max_streams) return fail(PB_ERR_INVALID, "bad n");
    if (n == 0) return PB_OK;
    if (!d_out) return fail(PB_ERR_INVALID, "null buffer");
    CK(cudaSetDevice(h->cfg.device));
    const K2In in = stream_k2in(h, d_ids);
    long long total = n * in.T * in.F_base;
    read_window_kernel<<<(int)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(in, d_ids, n, d_out);
    CK(cudaGetLastError());
    return PB_OK;
}

struct TrigArrays {
    int* trig[PB_MAX_MODELS];        // each bank model's TriggerDetector.activation; null past the last model
};

// With a history pool: the history of streams ids[i] (or i) restarts at their n_samples, so that no read returns audio of a
// stream's previous life.  Runs after whatever reset n_samples, on the same stream.
static int restart_history(pb_handle* h, const int32_t* d_ids, int64_t n, cudaStream_t s) {
    if (!h->history) return PB_OK;
    ProfScope ps(h, 3, s);
    history_restart_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(hist_pool(h), h->d_n_samples.get(), d_ids, n);
    CK(cudaGetLastError());
    return PB_OK;
}

// Stream ids[i] (or i) starts over: no samples consumed, every model's trigger re-armed.
__global__ void clear_kernel(long long* n_samples, TrigArrays t, const int* ids, long long n) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int sid = ids ? ids[i] : (int)i;
    n_samples[sid] = 0;
#pragma unroll
    for (int m = 0; m < PB_MAX_MODELS; ++m)
        if (t.trig[m]) t.trig[m][sid] = 0;
}

PB_API int pb_clear(pb_handle* h, const int32_t* d_ids, int64_t n, void* stream) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    if (n < 0 || n > h->cfg.max_streams) return fail(PB_ERR_INVALID, "bad n");
    if (n == 0) return PB_OK;
    CK(cudaSetDevice(h->cfg.device));
    TrigArrays t{};
    for (size_t m = 0; m < h->models.size(); ++m) t.trig[m] = h->models[m].trig.get();
    clear_kernel<<<(int)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(h->d_n_samples.get(), t, d_ids, n);
    CK(cudaGetLastError());
    if (h->pool) {
        pool_clear_kernel<<<(int)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(h->d_pool_trig.get(), d_ids, n);
        CK(cudaGetLastError());
    }
    return restart_history(h, d_ids, n, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------------
// per-stream model subscriptions

// Stream sids[j] gets mask masks[j]; every model m whose bit rearm[j] sets has its trigger re-armed for it.
__global__ void set_route_kernel(uint8_t* route, TrigArrays t, const int* sids, const uint8_t* masks, const uint8_t* rearm, long long k) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= k) return;
    const int sid = sids[j];
    route[sid] = masks[j];
#pragma unroll
    for (int m = 0; m < PB_MAX_MODELS; ++m)
        if (t.trig[m] && (rearm[j] >> m & 1)) t.trig[m][sid] = 0;
}

// The first pb_set_stream_models: device masks (every stream 0xFF), list scratch and its event.  Only then is the handle routed.
static int ensure_routed(pb_handle* h) {
    if (h->routed) return PB_OK;
    const size_t S = (size_t)h->cfg.max_streams;
    DevArray<uint8_t> route;
    DevArray<int2> lists;
    DevArray<unsigned> count;
    CK(route.alloc(S));
    CK(cudaMemset(route.get(), 0xFF, S));
    CK(lists.alloc(PB_MAX_MODELS * S));
    CK(count.alloc(PB_MAX_MODELS));
    CK(cudaEventCreateWithFlags(&h->route_ev, cudaEventDisableTiming));
    h->d_route = std::move(route);
    h->d_route_list = std::move(lists);
    h->d_route_count = std::move(count);
    h->route_mask.assign(S, 0xFF);
    for (int m = 0; m < PB_MAX_MODELS; ++m) h->subs[m] = (int64_t)S;
    h->routed = true;
    return PB_OK;
}

// Validates stream ids (h_ids null: 0..n-1) before anything changes: range and, for a set, uniqueness.
static int check_route_ids(const pb_handle* h, const int32_t* h_ids, int64_t n, bool unique) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    if (n < 0 || n > h->cfg.max_streams) return fail(PB_ERR_INVALID, "n = %lld outside [0, max_streams = %d]", (long long)n, h->cfg.max_streams);
    if (!h_ids) return PB_OK;
    std::vector<char> seen(unique ? h->cfg.max_streams : 0, 0);
    for (int64_t i = 0; i < n; ++i) {
        const int32_t sid = h_ids[i];
        if (sid < 0 || sid >= h->cfg.max_streams) return fail(PB_ERR_INVALID, "stream id %d outside [0, %d)", sid, h->cfg.max_streams);
        if (unique && seen[sid]++) return fail(PB_ERR_INVALID, "stream id %d appears twice", sid);
    }
    return PB_OK;
}

PB_API int pb_set_stream_models(pb_handle* h, const int32_t* h_ids, const uint8_t* h_masks, int64_t n) {
    int rc = check_route_ids(h, h_ids, n, true);
    if (rc != PB_OK) return rc;
    if (n > 0 && !h_masks) return fail(PB_ERR_INVALID, "null masks");
    CK(cudaSetDevice(h->cfg.device));
    rc = ensure_routed(h);
    if (rc != PB_OK) return rc;
    CK(cudaDeviceSynchronize());                     // queued work finishes under the old masks
    std::vector<int> sids;
    std::vector<uint8_t> masks, rearm;
    for (int64_t i = 0; i < n; ++i) {
        const int sid = h_ids ? h_ids[i] : (int)i;
        const uint8_t old = h->route_mask[sid], nw = h_masks[i];
        if (old == nw) continue;
        sids.push_back(sid);
        masks.push_back(nw);
        rearm.push_back((uint8_t)(nw & ~old));
    }
    if (sids.empty()) return PB_OK;
    DevArray<int> d_sids;
    DevArray<uint8_t> d_masks, d_rearm;
    CK(d_sids.upload(sids));
    CK(d_masks.upload(masks));
    CK(d_rearm.upload(rearm));
    TrigArrays t{};
    for (size_t m = 0; m < h->models.size(); ++m) t.trig[m] = h->models[m].trig.get();
    const long long k = (long long)sids.size();
    set_route_kernel<<<(int)((k + 255) / 256), 256>>>(h->d_route.get(), t, d_sids.get(), d_masks.get(), d_rearm.get(), k);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    for (size_t j = 0; j < sids.size(); ++j) {
        const uint8_t old = h->route_mask[sids[j]];
        for (int m = 0; m < PB_MAX_MODELS; ++m) h->subs[m] += (int)(masks[j] >> m & 1) - (int)(old >> m & 1);
        h->route_mask[sids[j]] = masks[j];
    }
    return PB_OK;
}

PB_API int pb_get_stream_models(const pb_handle* h, const int32_t* h_ids, int64_t n, uint8_t* h_masks) {
    const int rc = check_route_ids(h, h_ids, n, false);
    if (rc != PB_OK) return rc;
    if (n > 0 && !h_masks) return fail(PB_ERR_INVALID, "null masks");
    for (int64_t i = 0; i < n; ++i) h_masks[i] = h->routed ? h->route_mask[h_ids ? h_ids[i] : i] : 0xFF;
    return PB_OK;
}

// ------------------------------------------------------------------------------------------------
// per-stream TriggerDetector settings

static bool same_trig(const StreamTrig& a, const StreamTrig& b) {
    uint64_t x, y;
    memcpy(&x, &a.sensitivity, 8);
    memcpy(&y, &b.sensitivity, 8);
    return x == y && a.trigger_level == b.trigger_level && a.chunk_bytes == b.chunk_bytes;
}

// The first pb_set_stream_trigger on a model: its records, every stream on the model's defaults.  Only then is it flagged.
static int ensure_trig_records(pb_handle* h, Network& net) {
    if (net.trig_set) return PB_OK;
    const size_t S = (size_t)h->cfg.max_streams;
    const StreamTrig d = default_trig(net);
    DevArray<TrigRec> rec;
    CK(rec.upload(std::vector<TrigRec>(S, trig_record(d))));
    net.trig_rec = std::move(rec);
    net.trig_host.assign(S, d);
    net.trig_set = true;
    return PB_OK;
}

PB_API int pb_set_stream_trigger(pb_handle* h, int32_t slot, const int32_t* h_ids, const double* h_sensitivity,
                                 const int32_t* h_trigger_level, const int32_t* h_chunk_bytes, int64_t n) {
    int rc = check_route_ids(h, h_ids, n, true);
    if (rc != PB_OK) return rc;
    if (slot < 0 || slot >= (int)h->models.size()) return fail(PB_ERR_INVALID, "slot %d outside [0, %d)", slot, (int)h->models.size());
    if (n > 0 && (!h_sensitivity || !h_trigger_level || !h_chunk_bytes)) return fail(PB_ERR_INVALID, "null settings");
    for (int64_t i = 0; i < n; ++i)
        if (h_chunk_bytes[i] < 1)
            return fail(PB_ERR_INVALID, "chunk_bytes = %d (entry %lld) must be >= 1: TriggerDetector divides by it", h_chunk_bytes[i], (long long)i);
    CK(cudaSetDevice(h->cfg.device));
    CK(cudaDeviceSynchronize());                     // queued work finishes under the old settings
    Network& net = h->models[slot];
    rc = ensure_trig_records(h, net);
    if (rc != PB_OK) return rc;
    std::vector<int> sids;
    std::vector<StreamTrig> vals;
    std::vector<TrigRec> recs;
    for (int64_t i = 0; i < n; ++i) {
        const int sid = h_ids ? h_ids[i] : (int)i;
        const StreamTrig v{h_sensitivity[i], h_trigger_level[i], h_chunk_bytes[i]};
        if (same_trig(v, net.trig_host[sid])) continue;      // unchanged: the detector keeps its state
        sids.push_back(sid);
        vals.push_back(v);
        recs.push_back(trig_record(v));
    }
    if (sids.empty()) return PB_OK;
    DevArray<int> d_sids;
    DevArray<TrigRec> d_recs;
    CK(d_sids.upload(sids));
    CK(d_recs.upload(recs));
    const long long k = (long long)sids.size();
    set_trigger_kernel<<<(int)((k + 255) / 256), 256>>>(net.trig_rec.get(), net.trig.get(), d_sids.get(), d_recs.get(), k);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    for (size_t j = 0; j < sids.size(); ++j) net.trig_host[sids[j]] = vals[j];
    return PB_OK;
}

PB_API int pb_get_stream_trigger(const pb_handle* h, int32_t slot, const int32_t* h_ids, int64_t n, double* h_sensitivity,
                                 int32_t* h_trigger_level, int32_t* h_chunk_bytes) {
    const int rc = check_route_ids(h, h_ids, n, false);
    if (rc != PB_OK) return rc;
    if (slot < 0 || slot >= (int)h->models.size()) return fail(PB_ERR_INVALID, "slot %d outside [0, %d)", slot, (int)h->models.size());
    if (n > 0 && (!h_sensitivity || !h_trigger_level || !h_chunk_bytes)) return fail(PB_ERR_INVALID, "null output");
    const Network& net = h->models[slot];
    const StreamTrig d = default_trig(net);
    for (int64_t i = 0; i < n; ++i) {
        const StreamTrig& v = net.trig_set ? net.trig_host[h_ids ? h_ids[i] : i] : d;
        h_sensitivity[i] = v.sensitivity;
        h_trigger_level[i] = v.trigger_level;
        h_chunk_bytes[i] = v.chunk_bytes;
    }
    return PB_OK;
}

// ------------------------------------------------------------------------------------------------
// stream state export / import (stream_state.cuh)

static const char* const STATE_FIELD[] = {"magic", "version", "num_models", "sample_rate", "window_samples", "hop_samples",
                                          "n_fft", "n_filt", "n_mfcc", "n_features", "use_delta", "vectorizer"};
static_assert(sizeof(STATE_FIELD) / sizeof(STATE_FIELD[0]) == STATE_HEAD_WORDS, "one name per header word");

static StateLayout state_layout(const pb_handle* h) {
    const pb_config& c = h->cfg;
    const int32_t fe[] = {c.sample_rate, c.window_samples, c.hop_samples, c.n_fft, c.n_filt, c.n_mfcc, c.n_features,
                          c.use_delta, c.vectorizer};
    StateLayout L{};
    L.head[0] = PB_STATE_MAGIC;
    L.head[1] = PB_STATE_VERSION;
    L.head[2] = (unsigned)h->models.size();
    for (int i = 0; i < 9; ++i) L.head[3 + i] = (unsigned)fe[i];
    for (size_t m = 0; m < h->models.size(); ++m) L.trig[m] = h->models[m].trig.get();
    L.tail_vecs = h->tail_cap / 8;                                   // tail_cap is a multiple of 8 int16
    L.ring_vecs = h->ring_rows * h->row_stride / 4;                  // row_stride is a multiple of 4 floats
    L.rec_vecs = STATE_HEADER_VECS + L.tail_vecs + L.ring_vecs;
    return L;
}

PB_API int64_t pb_stream_state_bytes(const pb_handle* h) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    return state_layout(h).rec_vecs * 16;
}

PB_API int pb_export_streams(pb_handle* h, const int32_t* d_ids, int64_t n, void* d_out, void* stream) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    if (n < 0 || n > h->cfg.max_streams) return fail(PB_ERR_INVALID, "n = %lld outside [0, max_streams = %d]", (long long)n, h->cfg.max_streams);
    if (n == 0) return PB_OK;
    if (!d_out) return fail(PB_ERR_INVALID, "null d_out");
    if ((uintptr_t)d_out % 16 != 0) return fail(PB_ERR_INVALID, "d_out must be 16-byte aligned");
    CK(cudaSetDevice(h->cfg.device));
    const int per = STATE_THREADS / 32;
    export_state_kernel<<<(unsigned)((n + per - 1) / per), STATE_THREADS, 0, (cudaStream_t)stream>>>(
        state_layout(h), stream_state(h), d_ids, n, static_cast<uint4*>(d_out));
    CK(cudaGetLastError());
    if (h->pool) {                                   // a handle without a pool leaves pool_activation 0
        pool_state_kernel<true><<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
            h->d_pool_trig.get(), d_ids, n, static_cast<int*>(d_out), state_layout(h).rec_vecs * 4);
        CK(cudaGetLastError());
    }
    return PB_OK;
}

PB_API int pb_import_streams(pb_handle* h, const int32_t* h_ids, int64_t n, const void* d_in) {
    int rc = check_route_ids(h, h_ids, n, true);
    if (rc != PB_OK) return rc;
    if (n == 0) return PB_OK;
    if (!d_in) return fail(PB_ERR_INVALID, "null d_in");
    if ((uintptr_t)d_in % 16 != 0) return fail(PB_ERR_INVALID, "d_in must be 16-byte aligned");
    CK(cudaSetDevice(h->cfg.device));
    CK(cudaDeviceSynchronize());                     // queued work finishes on the old state
    const StateLayout L = state_layout(h);
    const uint4* in = static_cast<const uint4*>(d_in);
    DevArray<StateCheck> d_check;
    const StateCheck init{~0ull, 0u, 0u};
    CK(d_check.upload(std::vector<StateCheck>(1, init)));
    validate_state_kernel<<<(unsigned)((n + STATE_THREADS - 1) / STATE_THREADS), STATE_THREADS>>>(L, in, n, d_check.get());
    CK(cudaGetLastError());
    StateCheck chk;
    CK(cudaMemcpy(&chk, d_check.get(), sizeof(chk), cudaMemcpyDeviceToHost));
    if (chk.bad) {
        const long long i = (long long)(chk.first >> 8);
        const int reason = (int)(chk.first & 0xff);
        pb_stream_state_header hd;
        CK(cudaMemcpy(&hd, in + i * L.rec_vecs, sizeof(hd), cudaMemcpyDeviceToHost));
        if (reason == STATE_BAD_N_SAMPLES)
            return fail(PB_ERR_INVALID, "record %lld: n_samples = %lld < 0 (%u bad records; nothing imported)", i, (long long)hd.n_samples, chk.bad);
        unsigned got[STATE_HEAD_WORDS];
        memcpy(got, &hd, sizeof(got));
        const int k = reason - 1;
        if (k < 2)
            return fail(PB_ERR_INVALID, "record %lld: %s = 0x%x, expected 0x%x: not a stream state record of this format (%u bad records; nothing imported)",
                        i, STATE_FIELD[k], got[k], L.head[k], chk.bad);
        return fail(PB_ERR_INVALID, "record %lld: %s = %d, this handle has %d (%u bad records; nothing imported)", i, STATE_FIELD[k],
                    (int)got[k], (int)L.head[k], chk.bad);
    }
    // K1's aligned-only kernels (and k1 modes 2-6) need n_samples % 8 == 0 (§3 "Sticky routing"): an unaligned record makes the
    // handle ragged, as its first pb_update_ragged does
    if (chk.unaligned && h->k1_mode != 0)
        return fail(PB_ERR_STATE, "a record's n_samples is not a multiple of 8 (the stream took ragged ticks): it needs k1 mode 0; nothing imported");
    DevArray<int> d_sids;
    if (h_ids) CK(d_sids.upload(std::vector<int>(h_ids, h_ids + n)));
    const int per = STATE_THREADS / 32;
    import_state_kernel<<<(unsigned)((n + per - 1) / per), STATE_THREADS>>>(L, stream_state(h), d_sids.get(), n, in);
    CK(cudaGetLastError());
    if (h->pool) {                                   // the record's pool_activation; a handle without a pool ignores it
        pool_state_kernel<false><<<(unsigned)((n + 255) / 256), 256>>>(h->d_pool_trig.get(), d_sids.get(), n,
                                                                     static_cast<int*>(const_cast<void*>(d_in)), L.rec_vecs * 4);
        CK(cudaGetLastError());
    }
    rc = restart_history(h, d_sids.get(), n, 0);                   // history restarts at the record's n_samples
    if (rc != PB_OK) return rc;
    CK(cudaDeviceSynchronize());
    if (chk.unaligned) h->ragged = true;
    return PB_OK;
}

// ------------------------------------------------------------------------------------------------
// stream audio history (history.cuh)

PB_API int pb_set_history(pb_handle* h, int64_t history_samples, int32_t max_rows) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    const bool drop = history_samples == 0 && max_rows == 0;
    if (!drop) {
        if (history_samples < 1 || history_samples > INT32_MAX - 7)
            return fail(PB_ERR_INVALID, "history_samples = %lld outside [1, %d]", (long long)history_samples, INT32_MAX - 7);
        if (max_rows < 1 || max_rows > h->cfg.max_streams)
            return fail(PB_ERR_INVALID, "max_rows = %d outside [1, max_streams = %d]", max_rows, h->cfg.max_streams);
    }
    CK(cudaSetDevice(h->cfg.device));
    CK(cudaDeviceSynchronize());                     // queued ticks finish with the old pool
    h->history = false;                              // the old pool goes first, so a failed allocation leaves none
    h->d_hist = DevArray<int16_t>();
    h->d_hist_row = DevArray<int>();
    h->d_hist_start = DevArray<long long>();
    h->hist_row.clear();
    h->hist_free.clear();
    h->hist_samples = 0;
    h->hist_cap = h->hist_rows = 0;
    if (drop) return PB_OK;
    const size_t S = (size_t)h->cfg.max_streams;
    const int cap = (int)((history_samples + 7) & ~7LL);
    DevArray<int16_t> pool;
    DevArray<int> row_of;
    DevArray<long long> start;
    CK(pool.alloc((size_t)max_rows * cap));
    CK(row_of.alloc(S));
    CK(start.alloc(S));
    CK(cudaMemset(row_of.get(), 0xFF, S * sizeof(int)));
    CK(cudaMemset(start.get(), 0, S * sizeof(long long)));
    h->d_hist = std::move(pool);
    h->d_hist_row = std::move(row_of);
    h->d_hist_start = std::move(start);
    h->hist_row.assign(S, -1);
    for (int r = max_rows - 1; r >= 0; --r) h->hist_free.push_back(r);
    h->hist_samples = history_samples;
    h->hist_cap = cap;
    h->hist_rows = max_rows;
    h->history = true;
    return PB_OK;
}

PB_API int pb_set_stream_history(pb_handle* h, const int32_t* h_ids, const uint8_t* h_on, int64_t n) {
    int rc = check_route_ids(h, h_ids, n, true);
    if (rc != PB_OK) return rc;
    if (n > 0 && !h_on) return fail(PB_ERR_INVALID, "null h_on");
    if (!h->history) return fail(PB_ERR_STATE, "no history pool: call pb_set_history first");
    int64_t on_after = h->hist_rows - (int64_t)h->hist_free.size();
    for (int64_t i = 0; i < n; ++i) {
        const int sid = h_ids ? h_ids[i] : (int)i;
        on_after += (int)(h_on[i] != 0) - (int)(h->hist_row[sid] >= 0);
    }
    if (on_after > h->hist_rows)
        return fail(PB_ERR_INVALID, "%lld streams would have history, the pool has max_rows = %d; nothing changed", (long long)on_after,
                    h->hist_rows);
    CK(cudaSetDevice(h->cfg.device));
    CK(cudaDeviceSynchronize());                     // queued ticks finish with the old rows
    // rows of the streams that go off first, then one for each stream that goes on
    std::vector<int> free_rows = h->hist_free, sids, rows;
    for (int pass = 0; pass < 2; ++pass)
        for (int64_t i = 0; i < n; ++i) {
            const int sid = h_ids ? h_ids[i] : (int)i;
            const bool was = h->hist_row[sid] >= 0, on = h_on[i] != 0;
            if (pass == 0 && was && !on) {
                free_rows.push_back(h->hist_row[sid]);
                sids.push_back(sid);
                rows.push_back(-1);
            } else if (pass == 1 && !was && on) {
                sids.push_back(sid);
                rows.push_back(free_rows.back());
                free_rows.pop_back();
            }
        }
    if (sids.empty()) return PB_OK;
    DevArray<int> d_sids, d_rows;
    CK(d_sids.upload(sids));
    CK(d_rows.upload(rows));
    const long long k = (long long)sids.size();
    {
        ProfScope ps(h, 3, 0);
        history_set_kernel<<<(unsigned)((k + 255) / 256), 256>>>(hist_pool(h), h->d_n_samples.get(), d_sids.get(), d_rows.get(), k);
        CK(cudaGetLastError());
    }
    CK(cudaDeviceSynchronize());
    for (size_t j = 0; j < sids.size(); ++j) h->hist_row[sids[j]] = rows[j];
    h->hist_free = std::move(free_rows);
    return PB_OK;
}

PB_API int pb_get_stream_history(const pb_handle* h, const int32_t* h_ids, int64_t n, uint8_t* h_on) {
    const int rc = check_route_ids(h, h_ids, n, false);
    if (rc != PB_OK) return rc;
    if (n > 0 && !h_on) return fail(PB_ERR_INVALID, "null h_on");
    for (int64_t i = 0; i < n; ++i) h_on[i] = h->history && h->hist_row[h_ids ? h_ids[i] : i] >= 0;
    return PB_OK;
}

PB_API int pb_read_history(pb_handle* h, const int32_t* d_ids, int64_t n, int64_t samples, int16_t* d_out, void* stream) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    if (n < 0 || n > h->cfg.max_streams) return fail(PB_ERR_INVALID, "n = %lld outside [0, max_streams = %d]", (long long)n, h->cfg.max_streams);
    if (!h->history) return fail(PB_ERR_STATE, "no history pool: call pb_set_history first");
    if (samples < 1 || samples > h->hist_samples)
        return fail(PB_ERR_INVALID, "samples = %lld outside [1, history_samples = %lld]", (long long)samples, (long long)h->hist_samples);
    if (n == 0) return PB_OK;
    if (!d_out) return fail(PB_ERR_INVALID, "null d_out");
    CK(cudaSetDevice(h->cfg.device));
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope ps(h, 3, s);
    history_read_kernel<<<(unsigned)n, HIST_THREADS, 0, s>>>(hist_pool(h), h->d_n_samples.get(), d_ids, h->cfg.max_streams,
                                                              (int)samples, d_out);
    CK(cudaGetLastError());
    return PB_OK;
}

// ------------------------------------------------------------------------------------------------
// model pool (pool.cuh)

// Frees the pool, if any.  The device is the handle's and idle.
static void drop_pool(pb_handle* h) {
    h->pool = false;
    h->pool_models = 0;
    h->d_pool_slots = DevArray<uint4>();
    h->d_pool_count = DevArray<unsigned>();
    h->d_pool_list0 = DevArray<unsigned>();
    h->d_pool_id = DevArray<int>();
    h->d_pool_trig = DevArray<int>();
    h->d_pool_list = DevArray<int2>();
    for (int sh = 0; sh < 2; ++sh)
        for (int ka = 0; ka < 2; ++ka) { h->d_pool_tiles[sh][ka] = DevArray<int2>(); h->pool_tiles[sh][ka] = 0; }
    h->pool_id = std::vector<int>();
    h->pool_subs = std::vector<int64_t>();
    h->pool_keras = std::vector<uint8_t>();
    h->pool_cd_of.clear();
    h->pool_cd.clear();
    h->pool_cd_of.shrink_to_fit();
    h->pool_trig_set = false;
    h->pool_trig_host = std::vector<StreamTrig>();
    h->d_pool_trig_rec = DevArray<TrigRec>();
}

PB_API int pb_set_pool(pb_handle* h, int32_t max_models) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    if (max_models < 0 || max_models > (1 << 24)) return fail(PB_ERR_INVALID, "max_models = %d outside [1, 2^24] (0 frees the pool)", max_models);
    CK(cudaSetDevice(h->cfg.device));
    CK(cudaDeviceSynchronize());                     // queued ticks finish with the old pool
    drop_pool(h);                                    // the old pool goes first, so a failed allocation leaves none
    if (max_models == 0) return PB_OK;
    const size_t S = (size_t)h->cfg.max_streams, M = (size_t)max_models;
    DevArray<uint4> slots;
    DevArray<unsigned> count, list0;
    DevArray<int> id, trig;
    DevArray<int2> list;
    CK(slots.alloc(M * POOL_SLOT_U4));
    CK(count.alloc(M));
    CK(list0.alloc(M + 1));
    CK(id.alloc(S));
    CK(trig.alloc(S));
    CK(list.alloc(S));
    CK(cudaMemset(list0.get(), 0, (M + 1) * sizeof(unsigned)));
    CK(cudaMemset(id.get(), 0xFF, S * sizeof(int)));
    CK(cudaMemset(trig.get(), 0, S * sizeof(int)));
    CK(ensure_dyn_smem(pool_warp_kernel<true>, (size_t)(MMA_THREADS / 32) * BANK_MODEL_SMEM));
    CK(ensure_dyn_smem(pool_warp_kernel<false>, (size_t)(MMA_THREADS / 32) * BANK_MODEL_SMEM));
    // 4 CTAs of 56 832 B per SM need the largest shared-memory carveout
    CK(cudaFuncSetAttribute(pool_warp_kernel<true>, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
    CK(cudaFuncSetAttribute(pool_warp_kernel<false>, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
    if (!h->pool_ev) CK(cudaEventCreateWithFlags(&h->pool_ev, cudaEventDisableTiming));
    h->d_pool_slots = std::move(slots);
    h->d_pool_count = std::move(count);
    h->d_pool_list0 = std::move(list0);
    h->d_pool_id = std::move(id);
    h->d_pool_trig = std::move(trig);
    h->d_pool_list = std::move(list);
    h->pool_id.assign(S, -1);
    h->pool_subs.assign(M, 0);
    h->pool_keras.assign(M, 0);
    h->pool_cd_of.assign(M, h->pool_cd.end());
    h->pool_models = max_models;
    h->pool = true;
    return PB_OK;
}

// list0 and the four tile tables from the host's per-model stream counts: model m's list positions [0, subs[m]) as block
// tiles of 64, the rest as warp tiles of 16.  Synchronous; the device is idle.
static int pool_rebuild(pb_handle* h) {
    const int M = h->pool_models;
    std::vector<unsigned> list0((size_t)M + 1);
    std::vector<int2> tiles[2][2];
    unsigned at = 0;
    for (int m = 0; m < M; ++m) {
        list0[m] = at;
        const int64_t s = h->pool_subs[m];
        at += (unsigned)s;
        const int ka = h->pool_keras[m];
        const int64_t nb = h->pool_warp_only ? 0 : s / 64;
        for (int64_t p = 0; p < nb * 64; p += 64) tiles[0][ka].push_back(make_int2(m, (int)p));
        for (int64_t p = nb * 64; p < s; p += 16) tiles[1][ka].push_back(make_int2(m, (int)p));
    }
    list0[M] = at;
    CK(cudaMemcpy(h->d_pool_list0.get(), list0.data(), list0.size() * sizeof(unsigned), cudaMemcpyHostToDevice));
    for (int sh = 0; sh < 2; ++sh)
        for (int ka = 0; ka < 2; ++ka) {
            CK(h->d_pool_tiles[sh][ka].upload(tiles[sh][ka]));
            h->pool_tiles[sh][ka] = (int64_t)tiles[sh][ka].size();
        }
    return PB_OK;
}

PB_API int pb_pool_load(pb_handle* h, int32_t model_id, const pb_config* cfg, const float* kernel, const float* recurrent,
                        const float* bias, const float* dense_w, float dense_b, const double* cd, int64_t cd_len) {
    if (!h || !cfg || !kernel || !recurrent || !bias || !dense_w) return fail(PB_ERR_INVALID, "null argument");
    if (!h->pool) return fail(PB_ERR_STATE, "no model pool: call pb_set_pool first");
    if (model_id < 0 || model_id >= h->pool_models) return fail(PB_ERR_INVALID, "model_id %d outside [0, max_models = %d)", model_id, h->pool_models);
    const pb_config& c = *cfg;
    int rc = check_front_end(h, c);
    if (rc != PB_OK) return rc;
    rc = check_network(c);
    if (rc != PB_OK) return rc;
    Network net;                                     // the network's fields, decoder table and range
    net.cfg = c;
    net.cfg.max_streams = h->cfg.max_streams;
    if (!bank_fused(net, h->feat))
        return fail(PB_ERR_UNSUPPORTED, "the model pool holds networks of the fused family (hidden <= %d, feature size <= %d, no deltas); "
                    "this one has hidden = %d, feature size = %d", BANK_MAX_H, BANK_MAX_F, c.hidden, h->feat);
    build_cdf(net);
    if (cd && cd_len != (int64_t)net.cd.size()) return fail(PB_ERR_INVALID, "cdf length %lld != %zu", (long long)cd_len, net.cd.size());
    if (cd) memcpy(net.cd.data(), cd, cd_len * sizeof(double));
    Frag16 fr;
    build_frag16(fr, c.hidden, h->feat, kernel, recurrent, bias, dense_w);
    std::vector<uint4> slot;
    slot.reserve(POOL_SLOT_U4);
    slot.insert(slot.end(), fr.bf16.begin(), fr.bf16.end());
    slot.insert(slot.end(), fr.xf16.begin(), fr.xf16.end());
    std::vector<float> tail(fr.mb);
    tail.insert(tail.end(), fr.mw.begin(), fr.mw.end());
    const size_t tail_u4 = tail.size() * sizeof(float) / 16;
    slot.resize(slot.size() + tail_u4);
    memcpy(slot.data() + slot.size() - tail_u4, tail.data(), tail.size() * sizeof(float));
    if (slot.size() != (size_t)POOL_FRAG_U4) return fail(PB_ERR_INVALID, "pool slot layout");
    slot.resize(POOL_SLOT_U4, uint4{});             // the record goes behind the weights
    CK(cudaSetDevice(h->cfg.device));
    CK(cudaDeviceSynchronize());                     // queued ticks finish with the old model
    // the decoder table: an existing one with these bytes, else a new one (a failure here changes nothing)
    std::string key(reinterpret_cast<const char*>(net.cd.data()), net.cd.size() * sizeof(double));
    auto it = h->pool_cd.find(key);
    if (it == h->pool_cd.end()) {
        pb_handle::PoolCd fresh;
        CK(fresh.d.upload(net.cd));
        it = h->pool_cd.emplace(std::move(key), std::move(fresh)).first;
    }
    ++it->second.refs;
    uint4* frag = h->d_pool_slots.get() + (size_t)model_id * POOL_SLOT_U4;
    PoolModel rec{};
    rec.w.bfrag = frag;
    rec.w.xfrag = frag + 2 * MMA_NT * 32;
    rec.w.bias = reinterpret_cast<const float*>(frag + BANK_FRAG_U4);
    rec.w.wd = rec.w.bias + 72;
    rec.w.bd = dense_b;
    rec.w.act = c.activation;
    rec.w.ract = c.recurrent_activation;
    rec.dp = decode_params(net);
    rec.dp.cd = it->second.d.get();
    memcpy(slot.data() + POOL_FRAG_U4, &rec, sizeof(rec));
    const cudaError_t e = cudaMemcpy(frag, slot.data(), slot.size() * sizeof(uint4), cudaMemcpyHostToDevice);   // weights and record at once
    if (e != cudaSuccess) {
        if (--it->second.refs == 0) h->pool_cd.erase(it);
        return fail(PB_ERR_CUDA, "pool slot upload failed: %s", cudaGetErrorString(e));
    }
    auto& old = h->pool_cd_of[model_id];
    if (old != h->pool_cd.end() && --old->second.refs == 0) h->pool_cd.erase(old);
    old = it;
    const uint8_t keras = keras_act(net);
    const bool moved = keras != h->pool_keras[model_id];
    h->pool_keras[model_id] = keras;
    if (h->pool_subs[model_id] > 0) {                // a new runner for the streams on the slot: fresh detectors
        const long long S = h->cfg.max_streams;
        pool_rearm_model_kernel<<<(unsigned)((S + 255) / 256), 256>>>(h->d_pool_id.get(), h->d_pool_trig.get(), S, model_id);
        CK(cudaGetLastError());
        if (moved) {                                 // its tiles change activation class
            rc = pool_rebuild(h);
            if (rc != PB_OK) return rc;
        }
        CK(cudaDeviceSynchronize());
    }
    return PB_OK;
}

PB_API int pb_set_stream_pool(pb_handle* h, const int32_t* h_ids, const int32_t* h_models, int64_t n) {
    int rc = check_route_ids(h, h_ids, n, true);
    if (rc != PB_OK) return rc;
    if (n > 0 && !h_models) return fail(PB_ERR_INVALID, "null model ids");
    if (!h->pool) return fail(PB_ERR_STATE, "no model pool: call pb_set_pool first");
    for (int64_t i = 0; i < n; ++i) {
        const int32_t m = h_models[i];
        if (m < -1 || m >= h->pool_models)
            return fail(PB_ERR_INVALID, "model id %d (entry %lld) outside [-1, max_models = %d); nothing changed", m, (long long)i, h->pool_models);
        if (m >= 0 && h->pool_cd_of[m] == h->pool_cd.end())
            return fail(PB_ERR_INVALID, "pool slot %d (entry %lld) holds no model: pb_pool_load it first; nothing changed", m, (long long)i);
    }
    CK(cudaSetDevice(h->cfg.device));
    CK(cudaDeviceSynchronize());                     // queued ticks finish under the old assignments
    std::vector<int> sids, models;
    for (int64_t i = 0; i < n; ++i) {
        const int sid = h_ids ? h_ids[i] : (int)i;
        if (h->pool_id[sid] == h_models[i]) continue;    // unchanged: the detector keeps its state
        sids.push_back(sid);
        models.push_back(h_models[i]);
    }
    if (sids.empty()) return PB_OK;
    DevArray<int> d_sids, d_models;
    CK(d_sids.upload(sids));
    CK(d_models.upload(models));
    const long long k = (long long)sids.size();
    pool_set_kernel<<<(unsigned)((k + 255) / 256), 256>>>(h->d_pool_id.get(), h->d_pool_trig.get(), d_sids.get(), d_models.get(), k);
    CK(cudaGetLastError());
    for (size_t j = 0; j < sids.size(); ++j) {
        int& cur = h->pool_id[sids[j]];
        if (cur >= 0) --h->pool_subs[cur];
        if (models[j] >= 0) ++h->pool_subs[models[j]];
        cur = models[j];
    }
    rc = pool_rebuild(h);
    if (rc != PB_OK) return rc;
    CK(cudaDeviceSynchronize());
    return PB_OK;
}

PB_API int pb_get_stream_pool(const pb_handle* h, const int32_t* h_ids, int64_t n, int32_t* h_models) {
    const int rc = check_route_ids(h, h_ids, n, false);
    if (rc != PB_OK) return rc;
    if (n > 0 && !h_models) return fail(PB_ERR_INVALID, "null model ids");
    for (int64_t i = 0; i < n; ++i) h_models[i] = h->pool ? h->pool_id[h_ids ? h_ids[i] : i] : -1;
    return PB_OK;
}

PB_API int pb_debug_pool_tiles(pb_handle* h, int warp_only) {
    if (!h) return fail(PB_ERR_INVALID, "null handle");
    if (!h->pool) return fail(PB_ERR_STATE, "no model pool: call pb_set_pool first");
    CK(cudaSetDevice(h->cfg.device));
    CK(cudaDeviceSynchronize());
    h->pool_warp_only = warp_only != 0;
    const int rc = pool_rebuild(h);
    if (rc != PB_OK) return rc;
    CK(cudaDeviceSynchronize());
    return PB_OK;
}

// The network half of a pool tick: the route, then the block and warp tiles of both activation classes; with per-stream
// trigger settings, the scans write raw and conf only and pool_trigger_kernel follows them.
static int score_pool(pb_handle* h, const int32_t* d_ids, int64_t n, float* d_raw, double* d_conf, uint8_t* d_fired,
                      unsigned long long* d_count, cudaStream_t s) {
    PoolTick t{};
    t.pool_id = h->d_pool_id.get(); t.slots = h->d_pool_slots.get(); t.lists = h->d_pool_list.get();
    t.count = h->d_pool_count.get(); t.list0 = h->d_pool_list0.get();
    t.raw = d_raw; t.conf = d_conf; t.fired = d_fired; t.d_count = d_count; t.trig = h->d_pool_trig.get();
    PoolTrig pt{};
    if (h->pool_trig_set) {
        pt.ids = d_ids; pt.n = n; pt.pool_id = t.pool_id; pt.slots = t.slots;
        pt.conf = d_conf; pt.fired = d_fired; pt.d_count = d_count; pt.trig = t.trig; pt.rec = h->d_pool_trig_rec.get();
        t.fired = nullptr; t.d_count = nullptr; t.trig = nullptr;
    }
    const K2In in = stream_k2in(h, d_ids);
    ProfScope ps(h, 1, s);
    // the lists and counts are the handle's: a pool tick on another stream may still be reading them
    CK(cudaStreamWaitEvent(s, h->pool_ev, 0));
    // the event is recorded after the tick's work even when a launch fails, so the next tick orders itself after it
    auto launch = [&]() -> int {
        CK(cudaMemsetAsync(t.count, 0, (size_t)h->pool_models * sizeof(unsigned), s));
        pool_route_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(d_ids, n, t);
        CK(cudaGetLastError());
        constexpr int W = MMA_THREADS / 32;
        for (int ka = 0; ka < 2; ++ka) {
            const int64_t nb = h->pool_tiles[0][ka], nw = h->pool_tiles[1][ka];
            const int2* tb = h->d_pool_tiles[0][ka].get();
            const int2* tw = h->d_pool_tiles[1][ka].get();
            if (nb && ka) pool_block_kernel<true><<<(unsigned)nb, MMA_THREADS, BANK_MODEL_SMEM + BANK_STAGE_SMEM, s>>>(tb, t, in);
            else if (nb) pool_block_kernel<false><<<(unsigned)nb, MMA_THREADS, BANK_MODEL_SMEM + BANK_STAGE_SMEM, s>>>(tb, t, in);
            CK(cudaGetLastError());
            if (nw && ka) pool_warp_kernel<true><<<(unsigned)((nw + W - 1) / W), MMA_THREADS, W * BANK_MODEL_SMEM, s>>>(tw, nw, t, in);
            else if (nw) pool_warp_kernel<false><<<(unsigned)((nw + W - 1) / W), MMA_THREADS, W * BANK_MODEL_SMEM, s>>>(tw, nw, t, in);
            CK(cudaGetLastError());
        }
        if (h->pool_trig_set) {
            pool_trigger_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(pt);
            CK(cudaGetLastError());
        }
        return PB_OK;
    };
    const int rc = launch();
    const cudaError_t er = cudaEventRecord(h->pool_ev, s);
    if (rc != PB_OK) return rc;
    if (er != cudaSuccess) return fail(PB_ERR_CUDA, "cudaEventRecord failed: %s", cudaGetErrorString(er));
    return PB_OK;
}

PB_API int pb_update_pool(pb_handle* h, const int16_t* d_pcm, const int64_t* d_offsets, int64_t max_len, const int32_t* d_ids,
                          int64_t n, float* d_raw, double* d_conf, uint8_t* d_fired, unsigned long long* d_count, void* stream) {
    int rc = check_tick(h, d_pcm, n);
    if (rc != PB_OK) return rc;
    if (!d_conf) return fail(PB_ERR_INVALID, "null d_conf");
    if (d_offsets && max_len < 1) return fail(PB_ERR_INVALID, "max_len = %lld must be >= 1", (long long)max_len);
    if (!h->pool) return fail(PB_ERR_STATE, "no model pool: call pb_set_pool first");
    if (d_offsets && h->k1_mode != 0) return fail(PB_ERR_STATE, "ragged ticks run only with k1 mode 0");
    if (n == 0) return PB_OK;
    CK(cudaSetDevice(h->cfg.device));
    cudaStream_t s = (cudaStream_t)stream;
    if (d_offsets) {                                 // pb_update_ragged's K1
        h->ragged = true;
        rc = append_history(h, d_pcm, d_offsets, max_len, d_ids, n, s);
        if (rc == PB_OK) rc = launch_ragged_mfcc(h, d_pcm, d_offsets, max_len, d_ids, n, s);
    } else {                                         // pb_update's
        rc = tick_mfcc(h, d_pcm, d_ids, n, s);
    }
    if (rc != PB_OK) return rc;
    return score_pool(h, d_ids, n, d_raw, d_conf, d_fired, d_count, s);
}

PB_API int pb_update_all(pb_handle* h, const int16_t* d_pcm, const int64_t* d_offsets, int64_t max_len, const int32_t* d_ids,
                         int64_t n, float* d_raw, double* d_conf, uint8_t* d_fired, unsigned long long* d_counts,
                         unsigned long long* d_pool_count, void* stream) {
    int rc = check_tick(h, d_pcm, n);
    if (rc != PB_OK) return rc;
    if (!d_conf) return fail(PB_ERR_INVALID, "null d_conf");
    if (d_offsets && max_len < 1) return fail(PB_ERR_INVALID, "max_len = %lld must be >= 1", (long long)max_len);
    if (!h->pool) return fail(PB_ERR_STATE, "no model pool: call pb_set_pool first");
    if (!h->models[0].w) return fail(PB_ERR_STATE, "pb_load_weights has not been called");
    if (d_offsets && h->k1_mode != 0) return fail(PB_ERR_STATE, "ragged ticks run only with k1 mode 0");
    if (n == 0) return PB_OK;
    CK(cudaSetDevice(h->cfg.device));
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t M = (int64_t)h->models.size();
    // K1 and the bank exactly as pb_update_ragged (offsets) or pb_update_models (none) run them, then the pool into row M
    if (d_offsets) {
        h->ragged = true;
        rc = append_history(h, d_pcm, d_offsets, max_len, d_ids, n, s);
        if (rc == PB_OK) rc = launch_ragged_mfcc(h, d_pcm, d_offsets, max_len, d_ids, n, s);
        if (rc == PB_OK)
            rc = M == 1 ? score_model0(h, d_ids, n, d_raw, d_conf, d_fired, d_counts, s)
                        : score_bank(h, d_ids, n, d_raw, d_conf, d_fired, d_counts, s);
    } else {
        rc = tick_mfcc(h, d_pcm, d_ids, n, s);
        if (rc == PB_OK) rc = score_bank(h, d_ids, n, d_raw, d_conf, d_fired, d_counts, s);
    }
    if (rc != PB_OK) return rc;
    return score_pool(h, d_ids, n, d_raw ? d_raw + M * n : nullptr, d_conf + M * n, d_fired ? d_fired + M * n : nullptr,
                      d_pool_count, s);
}

// ------------------------------------------------------------------------------------------------
// per-stream pool TriggerDetector settings

// A stream that follows its model: (NaN, 0, 0) on the host, trigger_reset 0 on the device.
static StreamTrig pool_follow_trig() {
    return StreamTrig{std::numeric_limits<double>::quiet_NaN(), 0, 0};
}

PB_API int pb_set_stream_pool_trigger(pb_handle* h, const int32_t* h_ids, const double* h_sensitivity,
                                      const int32_t* h_trigger_level, const int32_t* h_chunk_bytes, int64_t n) {
    int rc = check_route_ids(h, h_ids, n, true);
    if (rc != PB_OK) return rc;
    if (n > 0 && (!h_sensitivity || !h_trigger_level || !h_chunk_bytes)) return fail(PB_ERR_INVALID, "null settings");
    for (int64_t i = 0; i < n; ++i)
        if (h_chunk_bytes[i] < 0)
            return fail(PB_ERR_INVALID, "chunk_bytes = %d (entry %lld) must be >= 0 (0: the model's own settings)", h_chunk_bytes[i], (long long)i);
    if (!h->pool) return fail(PB_ERR_STATE, "no model pool: call pb_set_pool first");
    CK(cudaSetDevice(h->cfg.device));
    CK(cudaDeviceSynchronize());                     // queued work finishes under the old settings
    if (!h->pool_trig_set) {                         // the first call: every stream follows its model
        const size_t S = (size_t)h->cfg.max_streams;
        DevArray<TrigRec> rec;
        CK(rec.upload(std::vector<TrigRec>(S, TrigRec{0.0, 0, 0})));
        h->d_pool_trig_rec = std::move(rec);
        h->pool_trig_host.assign(S, pool_follow_trig());
        h->pool_trig_set = true;
    }
    std::vector<int> sids;
    std::vector<StreamTrig> vals;
    std::vector<TrigRec> recs;
    for (int64_t i = 0; i < n; ++i) {
        const int sid = h_ids ? h_ids[i] : (int)i;
        const bool follow = h_chunk_bytes[i] == 0;
        const StreamTrig v = follow ? pool_follow_trig() : StreamTrig{h_sensitivity[i], h_trigger_level[i], h_chunk_bytes[i]};
        if (same_trig(v, h->pool_trig_host[sid])) continue;  // unchanged: the detector keeps its state
        sids.push_back(sid);
        vals.push_back(v);
        recs.push_back(follow ? TrigRec{0.0, 0, 0} : trig_record(v));
    }
    if (sids.empty()) return PB_OK;
    DevArray<int> d_sids;
    DevArray<TrigRec> d_recs;
    CK(d_sids.upload(sids));
    CK(d_recs.upload(recs));
    const long long k = (long long)sids.size();
    set_trigger_kernel<<<(int)((k + 255) / 256), 256>>>(h->d_pool_trig_rec.get(), h->d_pool_trig.get(), d_sids.get(), d_recs.get(), k);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    for (size_t j = 0; j < sids.size(); ++j) h->pool_trig_host[sids[j]] = vals[j];
    return PB_OK;
}

PB_API int pb_get_stream_pool_trigger(const pb_handle* h, const int32_t* h_ids, int64_t n, double* h_sensitivity,
                                      int32_t* h_trigger_level, int32_t* h_chunk_bytes) {
    const int rc = check_route_ids(h, h_ids, n, false);
    if (rc != PB_OK) return rc;
    if (n > 0 && (!h_sensitivity || !h_trigger_level || !h_chunk_bytes)) return fail(PB_ERR_INVALID, "null output");
    const StreamTrig d = pool_follow_trig();
    for (int64_t i = 0; i < n; ++i) {
        const StreamTrig& v = h->pool_trig_set ? h->pool_trig_host[h_ids ? h_ids[i] : i] : d;
        h_sensitivity[i] = v.sensitivity;
        h_trigger_level[i] = v.trigger_level;
        h_chunk_bytes[i] = v.chunk_bytes;
    }
    return PB_OK;
}

// ------------------------------------------------------------------------------------------------
PB_API int pb_host_alloc(void** out, uint64_t bytes) {
    if (!out) return fail(PB_ERR_INVALID, "null argument");
    CK(cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocDefault));
    return PB_OK;
}

PB_API int pb_host_free(void* p) {
    if (p) CK(cudaFreeHost(p));
    return PB_OK;
}

static int ensure_pipe(pb_handle* h) {
    if (h->pipe[0]) return PB_OK;
    const int64_t sb = std::min<int64_t>(HOST_SUB_BATCH, h->cfg.max_streams);
    for (int i = 0; i < HOST_PIPE; ++i) {
        CK(cudaStreamCreateWithFlags(&h->pipe[i], cudaStreamNonBlocking));
        CK(cudaEventCreateWithFlags(&h->pipe_ev[i], cudaEventDisableTiming));
        CK(h->d_stage_pcm[i].alloc(sb * h->cfg.chunk_samples));
        CK(h->d_stage_ids[i].alloc(sb));
        CK(h->d_stage_raw[i].alloc(sb));
        CK(h->d_stage_conf[i].alloc(sb));
        CK(h->d_stage_fired[i].alloc(sb));
    }
    CK(cudaHostAlloc((void**)&h->h_count_pinned, sizeof(unsigned long long), cudaHostAllocDefault));
    return PB_OK;
}

__global__ void iota_kernel(int* ids, int base, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) ids[i] = base + i;
}

PB_API int pb_update_host(pb_handle* h, const int16_t* h_pcm, const int32_t* h_ids, int64_t n, float* h_raw, double* h_conf,
                   uint8_t* h_fired, unsigned long long* h_count) {
    int rc = check_tick(h, h_pcm, n);
    if (rc != PB_OK) return rc;
    if (n == 0) { if (h_count) *h_count = 0; return PB_OK; }
    if (!h->models[0].w) return fail(PB_ERR_STATE, "pb_load_weights has not been called");
    if (!h_conf) return fail(PB_ERR_INVALID, "null h_conf");
    CK(cudaSetDevice(h->cfg.device));
    rc = ensure_pipe(h);
    if (rc != PB_OK) return rc;
    const int64_t sb = std::min<int64_t>(HOST_SUB_BATCH, h->cfg.max_streams);
    const int chunk = h->cfg.chunk_samples;
    // ---- latency path (BASELINE configs[4]): a handful of streams in pinned host memory.  With unified addressing the
    // kernels read the PCM and write the results through the mapped host pointers directly: two launches and one
    // synchronisation instead of three staged copies.
    if (n <= HOST_ZERO_COPY_MAX) {
        auto pinned = [](const void* p) {
            if (!p) return true;
            cudaPointerAttributes a;
            if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
            return a.type == cudaMemoryTypeHost;
        };
        if (pinned(h_pcm) && pinned(h_ids) && pinned(h_raw) && pinned(h_conf) && pinned(h_fired)) {
            *h->h_count_pinned = 0;
            rc = pb_update(h, h_pcm, h_ids, n, h_raw, h_conf, h_fired, h->h_count_pinned, h->pipe[0]);
            if (rc != PB_OK) return rc;
            CK(cudaStreamSynchronize(h->pipe[0]));
            if (h_count) *h_count = *h->h_count_pinned;
            return PB_OK;
        }
    }
    // the counter is zeroed on pipe 0; the other pipes wait for that, pipe 0 waits for them at the end,
    // so the whole tick costs one host synchronisation
    unsigned long long* d_count = h->d_count.get();
    CK(cudaMemsetAsync(d_count, 0, sizeof(unsigned long long), h->pipe[0]));
    // equal sub-batches: nothing overlaps the first sub-batch's upload (pipeline fill) or the last one's kernels and download
    // (drain), and for a given number of sub-batches the largest one is smallest when all are equal (16 400 streams: 8 224 +
    // 8 176 rather than 16 384 + 16); step <= sb, a multiple of 32 except when one sub-batch takes everything
    const int64_t n_sub = (n + sb - 1) / sb;
    const int64_t step = n_sub == 1 ? n : std::min(sb, ((n + n_sub - 1) / n_sub + 31) & ~(int64_t)31);
    const int used_pipes = (int)std::min<int64_t>(HOST_PIPE, (n + step - 1) / step);
    if (used_pipes > 1) {
        CK(cudaEventRecord(h->pipe_ev[0], h->pipe[0]));
        for (int i = 1; i < used_pipes; ++i) CK(cudaStreamWaitEvent(h->pipe[i], h->pipe_ev[0], 0));
    }
    int p = 0;
    for (int64_t off = 0; off < n; off += step, p = (p + 1) % HOST_PIPE) {
        const int64_t m = std::min(step, n - off);
        cudaStream_t s = h->pipe[p];
        int16_t* pcm = h->d_stage_pcm[p].get();
        int* ids = h->d_stage_ids[p].get();
        float* raw = h->d_stage_raw[p].get();
        double* conf = h->d_stage_conf[p].get();
        uint8_t* fired = h->d_stage_fired[p].get();
        CK(cudaMemcpyAsync(pcm, h_pcm + off * chunk, m * chunk * sizeof(int16_t), cudaMemcpyHostToDevice, s));
        if (h_ids) CK(cudaMemcpyAsync(ids, h_ids + off, m * sizeof(int), cudaMemcpyHostToDevice, s));
        else { iota_kernel<<<(int)((m + 255) / 256), 256, 0, s>>>(ids, (int)off, (int)m); CK(cudaGetLastError()); }
        rc = pb_update(h, pcm, ids, m, h_raw ? raw : nullptr, conf, h_fired ? fired : nullptr, d_count, s);
        if (rc != PB_OK) return rc;
        CK(cudaMemcpyAsync(h_conf + off, conf, m * sizeof(double), cudaMemcpyDeviceToHost, s));
        if (h_raw) CK(cudaMemcpyAsync(h_raw + off, raw, m * sizeof(float), cudaMemcpyDeviceToHost, s));
        if (h_fired) CK(cudaMemcpyAsync(h_fired + off, fired, m * sizeof(uint8_t), cudaMemcpyDeviceToHost, s));
    }
    for (int i = 1; i < used_pipes; ++i) {
        CK(cudaEventRecord(h->pipe_ev[i], h->pipe[i]));
        CK(cudaStreamWaitEvent(h->pipe[0], h->pipe_ev[i], 0));
    }
    CK(cudaMemcpyAsync(h->h_count_pinned, d_count, sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->pipe[0]));
    CK(cudaStreamSynchronize(h->pipe[0]));
    if (h_count) *h_count = *h->h_count_pinned;
    return PB_OK;
}

