/*
 * precise_b200.h -- C ABI of libprecise_b200.so: the H100 (sm_90a) implementation of the
 * Mycroft Precise streaming-inference hot path
 *
 *      int16 PCM -> MFCC -> GRU window scan + Dense + sigmoid -> threshold decode -> trigger
 *
 * Every entry point names the reference interface it stands in for (paths relative to the
 * mycroft-precise checkout, commit e1a635e).  The reference is pure Python and has no FFI for
 * this path; INTEGRATION.md shows the ctypes stubs a maintainer would add behind
 * precise.network_runner.Runner / Listener and precise_runner.Engine.
 *
 * Conventions
 *   - every function returns PB_OK (0) or a negative pb_status; nothing throws across the ABI;
 *     pb_last_error() returns a thread-local message for the last failure on this thread.
 *   - pointers named d_* are DEVICE pointers on the handle's device, h_* are HOST pointers.
 *     All buffers are caller-owned and not retained after the call returns (device work is
 *     ordered on `stream`; the caller keeps buffers alive until that stream reaches the work).
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).  Calls are
 *     asynchronous with respect to the host unless stated otherwise.
 *   - a handle is not re-entrant (the reference drives one Listener from one thread,
 *     runner/precise_runner/runner.py:232-243); distinct handles / devices are independent.
 *   - there is no CPU fallback: without a CUDA device every compute entry point fails with
 *     PB_ERR_CUDA.
 */
#ifndef PRECISE_B200_H
#define PRECISE_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PB_ABI_VERSION 2
#define PB_MAX_THRESHOLDS 8
#define PB_MAX_MODELS 8           /* networks a handle's model bank holds (pb_add_model), slot 0 included */

typedef enum pb_status {
    PB_OK = 0,
    PB_ERR_INVALID = -1,      /* bad argument / shape; maps to ValueError            */
    PB_ERR_UNSUPPORTED = -2,  /* legal in the reference, not implemented here        */
    PB_ERR_CUDA = -3,         /* CUDA runtime / driver failure; maps to RuntimeError */
    PB_ERR_STATE = -4,        /* call order (e.g. predict before load_weights)       */
    PB_ERR_EOF = -5           /* empty chunk; maps to EOFError (network_runner.py:133-134) */
} pb_status;

/* Vectorizer ids, precise/params.py:121-133 */
enum { PB_VEC_MELS = 1, PB_VEC_MFCCS = 2, PB_VEC_SPEECHPY_MFCCS = 3 /* legacy vectoriser (precise/vectorization.py:40-42); restated from speechpy's published algorithm, parity unpinned */ };
/* activations of the GRU layer (precise/model.py:77-82 uses linear + Keras default hard_sigmoid) */
enum { PB_ACT_LINEAR = 0, PB_ACT_TANH = 1 };
enum { PB_RACT_HARD_SIGMOID = 0, PB_RACT_SIGMOID = 1 };

/*
 * Mirrors precise.params.ListenerParams (precise/params.py:29-118, defaults :140-144) with the
 * time fields already converted to samples the way the reference's properties do
 * (window_samples :85-87, hop_samples :90-92, n_features :80-82), plus the network size
 * (precise/model.py:40 recurrent_units), the ThresholdDecoder arguments
 * (precise/threshold_decoder.py:38) and the TriggerDetector arguments
 * (runner/precise_runner/runner.py:121).
 */
typedef struct pb_config {
    int32_t abi_version;       /* must be PB_ABI_VERSION                                     */
    int32_t device;            /* CUDA device ordinal                                        */
    int32_t max_streams;       /* capacity of the per-stream state (>= 1)                    */
    int32_t chunk_samples;     /* int16 samples per update per stream (runner.py:23: 2048 B = 1024) */
    /* ---- ListenerParams ---- */
    int32_t sample_rate;       /* 16000 */
    int32_t window_samples;    /* 1600  */
    int32_t hop_samples;       /* 800   */
    int32_t n_fft;             /* 512; power of two in [64, 1024]                            */
    int32_t n_filt;            /* 20;  <= 64                                                 */
    int32_t n_mfcc;            /* 13;  <= 64                                                 */
    int32_t n_features;        /* 29 rows per network input                                  */
    int32_t use_delta;         /* 0                                                          */
    int32_t vectorizer;        /* PB_VEC_MFCCS                                               */
    /* ---- network ---- */
    int32_t hidden;            /* GRU units, 20                                              */
    int32_t activation;        /* PB_ACT_LINEAR                                              */
    int32_t recurrent_activation; /* PB_RACT_HARD_SIGMOID                                    */
    /* ---- ThresholdDecoder ---- */
    int32_t n_thresholds;      /* number of (mu, std) pairs, 1..PB_MAX_THRESHOLDS            */
    double threshold_mu[PB_MAX_THRESHOLDS];   /* 6.0 */
    double threshold_std[PB_MAX_THRESHOLDS];  /* 4.0 */
    double threshold_center;   /* 0.2 */
    /* ---- TriggerDetector ---- */
    double sensitivity;        /* 0.5 */
    int32_t trigger_level;     /* 3   */
    int32_t decode_legacy_f64; /* 0 (default): asigmoid's `1 / x - 1` in float32, what the reference computes for the
                                * np.float32 that Runner.run returns (network_runner.py:73-74, functions.py:99-101) under
                                * NumPy >= 2 scalar promotion -- the behaviour of the reference run in this image;
                                * 1: the same expression in float64, what NumPy 1.16 (the reference's own pin, setup.py:74)
                                * evaluates, because legacy promotion makes `1 / np.float32` a float64 */
} pb_config;

typedef struct pb_handle pb_handle;

/* Fills *cfg with the reference defaults (precise/params.py:140-144, precise/model.py:40,
 * runner/precise_runner/runner.py:121,167), max_streams = 1, device = 0. */
int pb_config_default(pb_config* cfg);

/* Replaces Listener.__init__ (precise/network_runner.py:101-109): allocates per-stream state
 * (tail PCM, MFCC ring, trigger counters) for cfg->max_streams streams on cfg->device, builds
 * the mel filterbank / DCT / twiddle / CDF tables.  Derived feature width
 * feature_size = (vectorizer == MELS ? n_filt : min(n_filt, n_mfcc)) * (use_delta ? 2 : 1)
 * (precise/params.py:100-109). */
int pb_create(const pb_config* cfg, pb_handle** out);
void pb_destroy(pb_handle* h);

/* Replaces model loading (precise/model.py:48-54, network_runner.py:50-57 / :85-86).  HOST
 * pointers, Keras layout and gate order z,r,h: kernel[F][3H], recurrent[H][3H], bias[3H],
 * dense_w[H], dense_b; F = feature_size.  Synchronous. */
int pb_load_weights(pb_handle* h, const float* h_kernel, const float* h_recurrent,
                    const float* h_bias, const float* h_dense_w, float dense_b);

/* Number of MFCC frames vectorize_raw() yields for n samples:
 * n < window ? 0 : (n - window) / hop + 1  (sonopy framing, precise/vectorization.py:36-39). */
int64_t pb_mfcc_frames(const pb_handle* h, int64_t samples_per_stream);
int32_t pb_feature_size(const pb_handle* h);     /* network input width incl. deltas           */
int32_t pb_mfcc_width(const pb_handle* h);       /* columns vectorize_raw() returns            */

/* K1, stateless.  Replaces buffer_to_audio + vectorize_raw (precise/util.py:35-37,
 * precise/vectorization.py:46-50) for n_streams independent buffers:
 *   d_pcm [n_streams][samples_per_stream] int16 (scaled by 1/32768 like buffer_to_audio)
 *   d_out [n_streams][pb_mfcc_frames()][pb_mfcc_width()] float32 */
int pb_mfcc(pb_handle* h, const int16_t* d_pcm, int64_t n_streams, int64_t samples_per_stream,
            float* d_out, void* stream);
/* Same for float32 samples that are already scaled (the ndarray branch of
 * Listener.update_vectors, network_runner.py:126-127, and load_audio, util.py:65). */
int pb_mfcc_f32(pb_handle* h, const float* d_audio, int64_t n_streams, int64_t samples_per_stream,
                float* d_out, void* stream);

/* K2(+sigmoid), stateless.  Replaces Runner.predict (network_runner.py:35-37, :69-71, :88-92):
 *   d_inputs [n][n_features][feature_size] float32 -> d_out [n] float32 (the [n,1] column).
 * d_logit (optional, may be NULL) receives the pre-sigmoid Dense output. */
int pb_predict(pb_handle* h, const float* d_inputs, int64_t n, float* d_out, float* d_logit,
               void* stream);

/* K3, stateless.  Replaces ThresholdDecoder.decode (threshold_decoder.py:45-57) element-wise:
 *   d_raw [n] float32 -> d_conf [n] float64. */
int pb_decode(pb_handle* h, const float* d_raw, int64_t n, double* d_conf, void* stream);

/* Stateful tick.  Replaces, for n streams at once, Listener.update (network_runner.py:148-153)
 * followed by TriggerDetector.update (runner.py:127-142):
 *   d_pcm        [n][chunk_samples] int16, row i belongs to stream d_stream_ids[i]
 *   d_stream_ids [n] int32 in [0, max_streams), unique; NULL means 0..n-1
 *   d_raw        [n] float32  network output (optional, may be NULL)
 *   d_conf       [n] float64  decoded confidence (what Listener.update returns)
 *   d_fired      [n] uint8    TriggerDetector.update result (optional, may be NULL)
 *   d_count      [1] uint64   += number of streams that fired this tick (optional; the
 *                             caller zeroes it; this is the quantity all-reduced across GPUs) */
int pb_update(pb_handle* h, const int16_t* d_pcm, const int32_t* d_stream_ids, int64_t n,
              float* d_raw, double* d_conf, uint8_t* d_fired, unsigned long long* d_count,
              void* stream);

/* Model bank: several networks scored per tick over the handle's one MFCC front end (e.g. a wake word and a wake-up word,
 * each a Listener + TriggerDetector of its own fed the same chunk).  Slot 0 is the handle's own network (pb_create /
 * pb_load_weights); pb_add_model appends slot 1, 2, ... up to PB_MAX_MODELS models in all.  Models cannot be removed.
 *
 * pb_add_model: cfg supplies the model's network (hidden, activation, recurrent_activation), ThresholdDecoder
 * (n_thresholds, threshold_mu / _std, threshold_center, decode_legacy_f64) and TriggerDetector (sensitivity, trigger_level)
 * fields.  Its front-end fields (sample_rate, window_samples, hop_samples, n_fft, n_filt, n_mfcc, n_features, use_delta,
 * vectorizer, chunk_samples, device) must equal the handle's, else PB_ERR_INVALID naming the field; max_streams is taken
 * from the handle.  Weights as pb_load_weights (HOST pointers, Keras layout).  h_cd (optional, may be NULL = the built-in
 * table) is the model's CDF table of cd_len entries, as pb_set_cdf takes it.  *slot (optional) receives the model's slot.
 * Allocates the weights, tables and a [max_streams] int32 trigger state; no second ring or tail.
 * Synchronous. */
int pb_add_model(pb_handle* h, const pb_config* cfg, const float* h_kernel, const float* h_recurrent,
                 const float* h_bias, const float* h_dense_w, float dense_b, const double* h_cd, int64_t cd_len,
                 int32_t* slot);
/* Number of models in the bank (>= 1), or a negative pb_status. */
int pb_num_models(const pb_handle* h);
/* Bank tick: the pb_update tick for every model of the bank, MFCC computed once.  Outputs are model-major, M = pb_num_models:
 *   d_raw [M][n] float32 (optional), d_conf [M][n] float64, d_fired [M][n] uint8 (optional),
 *   d_count [M] uint64 (optional; d_count[m] += streams model m fired for this tick).
 * d_pcm / d_stream_ids as pb_update.  PB_ERR_STATE if slot 0 has no weights. */
int pb_update_models(pb_handle* h, const int16_t* d_pcm, const int32_t* d_stream_ids, int64_t n,
                     float* d_raw, double* d_conf, uint8_t* d_fired, unsigned long long* d_count, void* stream);

/* Ragged tick: the pb_update_models tick, but stream i brings its own number of samples, as Listener.update takes a chunk of
 * any length (network_runner.py:125-153).  For every stream and bank model: Listener.update(chunk) then TriggerDetector.update.
 *   d_pcm        packed int16 samples; item i's chunk is d_pcm[d_offsets[i] .. d_offsets[i+1])
 *   d_offsets    [n+1] int64, DEVICE, non-decreasing; any alignment (odd offsets allowed); d_pcm holds at least
 *                d_offsets[n] samples
 *   max_len      host-side upper bound on every d_offsets[i+1] - d_offsets[i] (>= 1)
 *   d_stream_ids as pb_update; outputs model-major as pb_update_models ([M][n], d_count [M]).  A one-model handle scores
 *                as pb_update does ([1][n] is its layout), a bank as pb_update_models does.
 * Every length must lie in [1, max_len].  The kernels clamp lengths to [0, max_len] and never read outside
 * [d_pcm + d_offsets[0], d_pcm + d_offsets[n]), so a caller's mistake gives wrong answers for that stream, never an
 * out-of-bounds access.  A chunk may complete any number of MFCC frames (long chunks run as several MFCC launches).
 * TriggerDetector's refractory count does not follow the lengths: the reference fixes chunk_size when it builds the detector
 * (runner/precise_runner/runner.py:121, :140), whatever the lengths of later reads.  It comes from the handle's chunk_samples
 * unless pb_set_stream_trigger gives the stream the chunk size of its own runner.
 * After a handle's first ragged tick, its uniform ticks (pb_update, pb_update_models, pb_update_vectors, pb_update_host) run
 * the ragged tick's MFCC kernel too (a stream's sample count is then no longer a multiple of 8), and pb_debug_k1_mode accepts
 * only 0.
 * PB_ERR_INVALID: null handle, d_offsets or d_conf, n outside [0, max_streams], max_len < 1.  PB_ERR_STATE: slot 0 has no
 * weights, or pb_debug_k1_mode is non-zero. */
int pb_update_ragged(pb_handle* h, const int16_t* d_pcm, const int64_t* d_offsets, int64_t max_len,
                     const int32_t* d_stream_ids, int64_t n, float* d_raw, double* d_conf, uint8_t* d_fired,
                     unsigned long long* d_count, void* stream);

/* Listener.update_vectors only (network_runner.py:125-146): advance stream state, no network. */
int pb_update_vectors(pb_handle* h, const int16_t* d_pcm, const int32_t* d_stream_ids, int64_t n,
                      void* stream);

/* Same tick with HOST buffers (what Engine.get_prediction sees: runner.py:62-67).  Copies are
 * pipelined in sub-batches over internal streams; returns when h_conf/h_fired/h_count are
 * valid.  Pinned buffers (pb_host_alloc) are needed for full PCIe rate.  h_stream_ids may be
 * NULL; h_raw, h_fired, h_count may be NULL; *h_count receives this tick's count. */
int pb_update_host(pb_handle* h, const int16_t* h_pcm, const int32_t* h_stream_ids, int64_t n,
                   float* h_raw, double* h_conf, uint8_t* h_fired, unsigned long long* h_count);

/* The 29 x F window Listener.update_vectors returns (network_runner.py:146), gathered for the
 * given streams: d_out [n][n_features][pb_mfcc_width()] float32, oldest row first. */
int pb_read_window(pb_handle* h, const int32_t* d_stream_ids, int64_t n, float* d_out, void* stream);

/* Replaces Listener.clear (network_runner.py:121-123) and re-arms the stream's trigger counter (of every bank model, and its
 * pool detector).
 * d_stream_ids NULL => streams 0..n-1. */
int pb_clear(pb_handle* h, const int32_t* d_stream_ids, int64_t n, void* stream);

/* Per-stream model subscriptions, as a device of a many-streams server runs a Listener only for its own wake word(s).
 * Bit m of a stream's mask = bank slot m scores that stream.  Every stream starts with mask 0xFF: every model, including
 * models added later.  Bits at or above pb_num_models are stored and take effect when such a model is added.  HOST arrays;
 * h_stream_ids NULL => 0..n-1.  Synchronous: work already queued on the device finishes under the old masks.  A bit that goes
 * from 0 to 1 re-arms that model's TriggerDetector for that stream, as a new detector would start.  PB_ERR_INVALID (and
 * nothing changes): null handle, n outside [0, max_streams], an id outside [0, max_streams), a duplicate id.
 *
 * pb_update, pb_update_host (bit 0), pb_update_models and pb_update_ragged honour the masks.  For a (stream item, model) pair
 * whose bit is clear: raw and conf are NaN, fired is 0, the model's trigger state for that stream does not change and nothing
 * is added to its count.  A stream with mask 0 still advances its MFCC state (pb_read_window sees its real window).
 * pb_clear leaves masks as they are.  A bank tick costs one window scan per subscribed (stream, model) pair; K1 and the ring
 * stay shared.  A handle that never calls pb_set_stream_models runs exactly as before; the first call allocates
 * [max_streams] mask bytes and 64 B per stream of route-list scratch.  Two bank ticks of one routed handle on different CUDA
 * streams are ordered by the library (they share that scratch). */
int pb_set_stream_models(pb_handle* h, const int32_t* h_stream_ids, const uint8_t* h_masks, int64_t n);
/* The masks of the given streams (h_stream_ids NULL => 0..n-1) into h_masks [n] (HOST).  PB_ERR_INVALID: null handle, n outside
 * [0, max_streams], an id outside [0, max_streams). */
int pb_get_stream_models(const pb_handle* h, const int32_t* h_stream_ids, int64_t n, uint8_t* h_masks);

/* Per-stream TriggerDetector settings of bank slot `slot`, as TriggerDetector(chunk_size, sensitivity, trigger_level)
 * (runner/precise_runner/runner.py:121) with each device's own values: Mycroft sets sensitivity and trigger_level per wake
 * word in each device's configuration, and each runner reads its own chunk_size.  HOST arrays of n entries; h_stream_ids
 * NULL => 0..n-1.  chunk_bytes is the runner's chunk_size in BYTES (refractory = -(8*2048) // chunk_bytes, Python floor
 * division).
 *   - Defaults: a stream never set uses the model's cfg.sensitivity, cfg.trigger_level and 2 * chunk_samples;
 *     pb_get_stream_trigger returns those for it, and exactly what was set (the sensitivity bit for bit) for a stream set.
 *   - Comparison: a tick compares conf > 1.0 - sensitivity in double (runner.py:130).  Any double is accepted (NaN and
 *     values outside [0, 1] included, as Python accepts them), any int32 trigger_level; chunk_bytes must be >= 1 (the
 *     reference would raise ZeroDivisionError).
 *   - Re-arming: an entry whose values change re-arms that model's detector for that stream (activation 0), as Mycroft
 *     builds a new runner when a setting changes; an entry set to the values it already has keeps its state.
 *   - PB_ERR_INVALID, and nothing changes: null handle, slot outside [0, pb_num_models), n outside [0, max_streams], an id
 *     outside [0, max_streams), a duplicate id, chunk_bytes < 1, a null array with n > 0.
 *   - Synchronous: work already queued on the device finishes under the old settings.
 *   - pb_clear re-arms a stream's detectors and keeps its settings; subscription changes (pb_set_stream_models) keep them
 *     too, and a mask bit going from 0 to 1 still re-arms.
 *   - pb_update, pb_update_host (zero-copy and pipelined), pb_update_models and pb_update_ragged honour the settings, with
 *     or without subscriptions; unsubscribed pairs stay NaN / NaN / 0 and their detector does not move.
 *   - Storage: the first call on a slot allocates that model's records, 16 B per stream on the device (initialised to the
 *     model's defaults) and a 16 B host mirror, and flags the model for good: its ticks then scan without the trigger and
 *     run one trigger kernel afterwards.  A model never set runs as before.  pb_destroy releases the records.
 *   - pb_add_model after settings exist: the new slot starts on its own defaults. */
int pb_set_stream_trigger(pb_handle* h, int32_t slot, const int32_t* h_stream_ids, const double* h_sensitivity,
                          const int32_t* h_trigger_level, const int32_t* h_chunk_bytes, int64_t n);
/* The settings of the given streams (h_stream_ids NULL => 0..n-1) of slot `slot` into h_sensitivity / h_trigger_level /
 * h_chunk_bytes [n] (HOST).  PB_ERR_INVALID: null handle or output with n > 0, bad slot, n outside [0, max_streams], an id
 * outside [0, max_streams). */
int pb_get_stream_trigger(const pb_handle* h, int32_t slot, const int32_t* h_stream_ids, int64_t n,
                          double* h_sensitivity, int32_t* h_trigger_level, int32_t* h_chunk_bytes);

/* Stream state export / import: a stream's listener state (Listener's window_audio and mfccs, network_runner.py:101-109,
 * and each bank model's TriggerDetector.activation, runner.py:125) as a self-describing record, so a stream can be
 * checkpointed to host memory or disk, or moved to another handle (a larger max_streams, another GPU, a new process).
 *
 * Record layout, pb_stream_state_bytes(h) bytes, every section 16-byte aligned:
 *   [0, 96)                      pb_stream_state_header below
 *   [96, 96 + 2 tail_cap)        the tail, tail_cap int16 copied whole; tail_cap = round_up(min(n_fft, window_samples), 8)
 *   [96 + 2 tail_cap, end)       the MFCC ring, ring_rows x row_stride float32 copied whole, padding columns included;
 *                                row_stride = round_up(mfcc width, 4), ring_rows = n_features + (release window - min(n_fft,
 *                                window_samples)) / hop_samples + 2, release window = window_samples (+ hop_samples for the
 *                                speechpy vectoriser)
 * The size depends only on the front-end fields, so two handles with the same front end agree on it (1024 + 2048 + 96 =
 * 3168 B at the defaults).  Not in the record: subscription masks and per-stream trigger settings (pb_get_stream_models /
 * pb_get_stream_trigger read them), the stream's pool model (pb_get_stream_pool), and the handle's chunk_samples (a record
 * imports into a handle with another chunk).  A handle with a model pool writes the stream's pool detector into pool_activation
 * and reads it back on import; a handle without one writes 0 and ignores it. */
#define PB_STATE_MAGIC 0x53534250u    /* "PBSS" in little-endian bytes */
#define PB_STATE_VERSION 1
typedef struct pb_stream_state_header {
    uint32_t magic;                   /* PB_STATE_MAGIC                                                     */
    uint32_t version;                 /* PB_STATE_VERSION                                                   */
    int32_t num_models;               /* pb_num_models of the exporting handle                              */
    int32_t sample_rate, window_samples, hop_samples, n_fft, n_filt, n_mfcc, n_features, use_delta, vectorizer;
    int64_t n_samples;                /* samples the stream has consumed                                    */
    int32_t pool_activation;          /* TriggerDetector.activation of the stream's pool model; 0 without a pool */
    int32_t reserved;                 /* 0                                                                  */
    int32_t activation[PB_MAX_MODELS];  /* TriggerDetector.activation of bank slot m; 0 from num_models on  */
} pb_stream_state_header;

/* Bytes of one stream's record (a multiple of 16), or a negative pb_status. */
int64_t pb_stream_state_bytes(const pb_handle* h);
/* Writes the records of streams d_stream_ids[i] (DEVICE; NULL => 0..n-1) to d_out [n][pb_stream_state_bytes] (DEVICE,
 * 16-byte aligned).  Asynchronous on `stream`, like pb_read_window: the caller orders it after the ticks whose state it
 * wants.  Reads state only: ticks after an export compute what they would have computed without it.  PB_ERR_INVALID: null
 * handle, n outside [0, max_streams], a null or unaligned d_out with n > 0. */
int pb_export_streams(pb_handle* h, const int32_t* d_stream_ids, int64_t n, void* d_out, void* stream);
/* Overwrites the state of streams h_stream_ids[i] (HOST; NULL => 0..n-1; unique, in [0, max_streams)) with record i of d_in
 * [n][pb_stream_state_bytes] (DEVICE, 16-byte aligned).  Slot m's activation goes to slot m: the caller makes sure the banks
 * correspond (the library does not fingerprint weights).  Synchronous: work already queued on the device finishes first.
 * Every record is validated before anything is written; on an error the handle is unchanged.
 *   PB_ERR_INVALID: null handle, n outside [0, max_streams], a bad or duplicate id, a null or unaligned d_in with n > 0, or a
 *   record with the wrong magic or version, a front-end field or model count that differs from this handle's, or
 *   n_samples < 0 (the message names the first bad record and the field).
 *   A record whose n_samples is not a multiple of 8 (a stream that took ragged ticks) makes the handle ragged, as its first
 *   pb_update_ragged does; PB_ERR_STATE if pb_debug_k1_mode is then non-zero.  Records that are all multiples of 8 leave
 *   the handle as it was, so its uniform ticks keep the fast MFCC kernel.
 * The imported streams keep this handle's masks and trigger settings. */
int pb_import_streams(pb_handle* h, const int32_t* h_stream_ids, int64_t n, const void* d_in);

/* Stream audio history: the recent int16 audio of chosen streams, kept on the device, so that a server can save the clip
 * behind an activation (the reference's listen.py keeps `audio_buffer`, buffer_samples long, and saves it on every
 * activation: precise/scripts/listen.py:59, :88-90).  Opt-in per stream: 2 B per sample and stream that has it.
 *   - Invariant: sample k of a stream's audio, counted as n_samples counts, lives at position k mod cap of the stream's row;
 *     cap is history_samples rounded up to a multiple of 8.  A chunk longer than cap keeps its last cap samples.
 *   - Which ticks append: every tick that consumes audio -- pb_update, pb_update_models, pb_update_ragged (each item's chunk
 *     exactly as K1 takes it, offsets clamped the same way), pb_update_vectors and pb_update_host (pipelined and zero-copy) --
 *     masks or not.  The stateless calls (pb_mfcc*, pb_predict) do not.
 *   - History start: a stream's n_samples when it was switched on, cleared (pb_clear: 0) or imported into (the record's
 *     n_samples), whichever came last.  Positions before it read as 0, so a read never returns audio of a previous life.
 *   - Not in state records (pb_export_streams): an imported stream that has history starts empty at the record's n_samples.
 *   - A handle without a pool runs exactly as before.
 *
 * pb_set_history: a pool of max_rows rows (max_rows in [1, max_streams]) of the last history_samples (>= 1) samples each.
 * Synchronous.  Calling it again replaces the pool and switches every stream off; (0, 0) frees it (pb_destroy frees it too).
 * PB_ERR_INVALID: null handle, a value out of range.  PB_ERR_CUDA: the allocation failed (the handle then has no pool). */
int pb_set_history(pb_handle* h, int64_t history_samples, int32_t max_rows);
/* Switches streams h_stream_ids[i] (HOST; NULL => 0..n-1) on (h_on[i] != 0) or off.  A stream that goes on starts empty at
 * its n_samples; one already on keeps its audio; one that goes off returns its row to the pool.  Validates everything before
 * it changes anything, then synchronises the device.  PB_ERR_INVALID, and nothing changes: null handle, n outside
 * [0, max_streams], an id outside [0, max_streams), a duplicate id, a null array with n > 0, more streams on than max_rows
 * after the call.  PB_ERR_STATE: no pool. */
int pb_set_stream_history(pb_handle* h, const int32_t* h_stream_ids, const uint8_t* h_on, int64_t n);
/* 1 if stream h_stream_ids[i] (HOST; NULL => 0..n-1) has history, else 0 (all 0 without a pool), into h_on [n] (HOST).
 * PB_ERR_INVALID: null handle or h_on with n > 0, n outside [0, max_streams], an id outside [0, max_streams). */
int pb_get_stream_history(const pb_handle* h, const int32_t* h_stream_ids, int64_t n, uint8_t* h_on);
/* d_out [n][samples] int16 (DEVICE): row i = samples [N - samples, N) of stream d_stream_ids[i] (DEVICE; NULL => 0..n-1),
 * oldest first, N = its n_samples at that point in stream order; 0 before its history start, all 0 for a stream that is off.
 * samples in [1, history_samples].  Asynchronous on `stream`, like pb_read_window; writes nothing but d_out.
 * PB_ERR_INVALID: null handle or d_out with n > 0, n outside [0, max_streams], samples out of range.  PB_ERR_STATE: no
 * pool. */
int pb_read_history(pb_handle* h, const int32_t* d_stream_ids, int64_t n, int64_t samples, int16_t* d_out, void* stream);

/* Model pool: a second, large set of networks on a handle, beside the bank, for a server whose devices each bring their own
 * wake word (custom models trained with precise-train, each used by one or a few devices).  Each stream points at at most one
 * pool model, or at none.  A pool tick runs K1 once, as every tick does, then scores every item whose stream has a pool model
 * with that model's network, ThresholdDecoder and TriggerDetector (the model's sensitivity and trigger_level, and the
 * refractory count from the handle's chunk_samples, unless pb_set_stream_pool_trigger gives the stream its own).  One window scan per item, whatever the number of models: the scan of a model
 * costs one 14 208 B weight load per tile of 64 (or of at most 16) of its streams.
 *   - Networks: the fused family only (hidden <= 24, feature size <= 16, no deltas), which every network precise-train builds
 *     at its defaults is in.  A pool stream's raw and conf are bit-identical to the same network's in a bank.
 *   - Memory: about 14.3 KB per slot, 51 200 B per distinct decoder table at the default thresholds (models whose tables
 *     are bit-identical share one copy), 16 B per stream.
 *   - The bank, its masks and trigger settings are independent of the pool; pb_update_models does not score pool models and
 *     pb_update_pool scores no bank model.  pb_update_all scores both on one K1.  pb_score_corpus scores the bank only;
 *     pb_score_corpus_pool scores chosen pool models over a recorded corpus, pb_score_corpus_pairs chosen (pool model,
 *     recording) pairs.  Not covered: pb_update_host, networks outside
 *     the fused family.
 *   - A handle that never calls pb_set_pool runs exactly as before.
 *
 * pb_set_pool: a pool of max_models slots (max_models in [1, 2^24]), every slot empty and every stream on none.  Synchronous.
 * Calling it again replaces the pool and unassigns every stream; 0 frees it (pb_destroy frees it too).  PB_ERR_INVALID: null
 * handle, max_models out of range.  PB_ERR_CUDA: an allocation failed (the handle then has no pool). */
int pb_set_pool(pb_handle* h, int32_t max_models);
/* Loads a network into slot model_id in [0, max_models): cfg, weights, h_cd and cd_len as pb_add_model takes them (front-end
 * fields equal to the handle's).  A slot that holds a model is replaced; its streams keep the slot and get fresh detectors, as
 * Mycroft builds a new runner for a new model, and score the new weights from the next tick.  Synchronous (queued work
 * finishes with the old model); on an error the slot is as it was.  PB_ERR_INVALID: a null argument, model_id out of range, a
 * front-end field that differs, a bad network field or cd_len.  PB_ERR_UNSUPPORTED: a network outside the fused family.
 * PB_ERR_STATE: no pool. */
int pb_pool_load(pb_handle* h, int32_t model_id, const pb_config* cfg, const float* h_kernel, const float* h_recurrent,
                 const float* h_bias, const float* h_dense_w, float dense_b, const double* h_cd, int64_t cd_len);
/* Stream h_stream_ids[i] (HOST; NULL => 0..n-1) goes to pool slot h_model_ids[i] (HOST), -1 = none.  Validates everything
 * before it changes anything, then synchronises the device.  A stream whose model changes gets a fresh detector; one set to
 * the model it has keeps its state.  pb_clear re-arms a stream's pool detector and keeps its model.  PB_ERR_INVALID, and
 * nothing changes: null handle, n outside [0, max_streams], an id outside [0, max_streams), a duplicate id, a null array with
 * n > 0, a model id outside [-1, max_models) or a slot that holds no model.  PB_ERR_STATE: no pool. */
int pb_set_stream_pool(pb_handle* h, const int32_t* h_stream_ids, const int32_t* h_model_ids, int64_t n);
/* The pool models of the given streams (h_stream_ids NULL => 0..n-1; -1 = none, and -1 for every stream without a pool) into
 * h_model_ids [n] (HOST).  PB_ERR_INVALID: null handle or output with n > 0, n outside [0, max_streams], an id outside
 * [0, max_streams). */
int pb_get_stream_pool(const pb_handle* h, const int32_t* h_stream_ids, int64_t n, int32_t* h_model_ids);
/* Pool tick.  d_offsets NULL: pb_update's uniform tick (d_pcm [n][chunk_samples], max_len ignored); otherwise pb_update_ragged's
 * (d_offsets [n+1] DEVICE, max_len >= 1, and the handle becomes ragged).  History is appended as on every tick.  Outputs are
 * [n]: d_raw (optional), d_conf, d_fired (optional), d_count [1] (optional, += the tick's pool fires).  An item whose stream
 * has no pool model gets NaN / NaN / 0; its detector does not move and it is not counted.  Needs no slot-0 weights.
 * d_stream_ids must be unique, as for pb_update; ids that repeat a stream give wrong answers for it but never a write outside
 * the pool's buffers (items past a model's stream count are not scored and get NaN / NaN / 0).
 * Asynchronous on `stream`; pool ticks on different CUDA streams are ordered by the library (they share list scratch).
 * PB_ERR_INVALID: null handle or d_conf, n outside [0, max_streams], max_len < 1 with offsets.  PB_ERR_STATE: no pool, or
 * offsets with a non-zero pb_debug_k1_mode. */
int pb_update_pool(pb_handle* h, const int16_t* d_pcm, const int64_t* d_offsets, int64_t max_len,
                   const int32_t* d_stream_ids, int64_t n, float* d_raw, double* d_conf, uint8_t* d_fired,
                   unsigned long long* d_count, void* stream);
/* Combined tick: the bank and the pool on one chunk, for a stream that listens for shared bank words and for its own pool
 * word.  d_offsets NULL: pb_update_models's uniform tick (d_pcm [n][chunk_samples], max_len ignored); otherwise
 * pb_update_ragged's (and the handle becomes ragged).  The tick appends history once and runs K1 once, then the bank's network
 * half exactly as pb_update_models / pb_update_ragged choose it (one model on a ragged tick: pb_update's path), then the pool's,
 * all on `stream`.  Outputs are [(M + 1)][n] for M = pb_num_models: rows 0 .. M-1 are bit-identical to what
 * pb_update_models / pb_update_ragged writes on a handle with the same bank, streams and audio (masks, NaN fill and per-stream
 * trigger settings included); row M to what pb_update_pool writes on a handle with the same pool (NaN / NaN / 0 for a stream
 * with no pool model).  d_raw and d_fired are optional.  d_counts [M] (optional) += each bank model's fires, d_pool_count [1]
 * (optional) += the pool's.  Ordering across CUDA streams as for the two ticks it combines.  Every argument is checked before
 * anything is enqueued, so a refused call changes no state.  PB_ERR_INVALID: as pb_update_ragged / pb_update_pool.
 * PB_ERR_STATE: no pool, slot 0 without weights, offsets with a non-zero pb_debug_k1_mode. */
int pb_update_all(pb_handle* h, const int16_t* d_pcm, const int64_t* d_offsets, int64_t max_len, const int32_t* d_stream_ids,
                  int64_t n, float* d_raw, double* d_conf, uint8_t* d_fired, unsigned long long* d_counts,
                  unsigned long long* d_pool_count, void* stream);
/* Per-stream TriggerDetector settings of the streams' pool models, as pb_set_stream_trigger sets them for a bank slot: stream
 * h_stream_ids[i] (HOST; NULL => 0..n-1) is scored by TriggerDetector(h_chunk_bytes[i], h_sensitivity[i],
 * h_trigger_level[i]), whichever pool model it is on.  The settings belong to the stream, not to a model.
 *   - Refractory count -(8*2048) // chunk_bytes (Python floor division).  chunk_bytes == 0 returns the stream to its model's
 *     own values (cfg.sensitivity, cfg.trigger_level, and the refractory count from the handle's chunk_samples), the state of
 *     a stream never set.  pb_get_stream_pool_trigger returns (NaN, 0, 0) for such a stream, otherwise exactly what was set
 *     (the sensitivity bit for bit); (NaN, 0, 0) for every stream without a pool.
 *   - A stream whose entry changes gets a fresh pool detector; an unchanged entry keeps it.  Settings survive
 *     pb_set_stream_pool (a changed model still re-arms), pb_pool_load and pb_clear; pb_set_pool (replace or free) drops them.
 *     pb_update_pool and pb_update_all honour them.
 *   - Validates everything before it changes anything, then synchronises the device.  PB_ERR_INVALID: null handle, n outside
 *     [0, max_streams], an id outside [0, max_streams), a duplicate id, a null array with n > 0, chunk_bytes < 0.
 *     PB_ERR_STATE: no pool.
 *   - Cost: the first call allocates a [max_streams] 16 B record array and a host mirror and flags the pool until it is
 *     replaced: its ticks then scan without the trigger and run one pool_trigger_kernel afterwards.  A pool never set runs as
 *     before. */
int pb_set_stream_pool_trigger(pb_handle* h, const int32_t* h_stream_ids, const double* h_sensitivity,
                               const int32_t* h_trigger_level, const int32_t* h_chunk_bytes, int64_t n);
/* The pool trigger settings of the given streams (h_stream_ids NULL => 0..n-1) into h_sensitivity / h_trigger_level /
 * h_chunk_bytes [n] (HOST).  PB_ERR_INVALID: null handle or output with n > 0, n outside [0, max_streams], an id outside
 * [0, max_streams). */
int pb_get_stream_pool_trigger(const pb_handle* h, const int32_t* h_stream_ids, int64_t n, double* h_sensitivity,
                               int32_t* h_trigger_level, int32_t* h_chunk_bytes);

/* Recorded corpora: whole recordings scored on the device in one call, the hot path of precise-simulate
 * (precise/scripts/simulate.py:92-129) and of false-activation mining (precise/scripts/train_incremental.py:113-137).
 * No stream state is read or written (n_samples, tails, rings, trigger state, history); subscriptions and per-stream trigger
 * settings do not apply.
 *
 * Schedules, for chunk c:
 *   PB_CORPUS_LISTENER  window k (k < floor(L / c)) is what Listener.update returns after samples [0, (k + 1) c) were fed in
 *                       chunks of c to a fresh listener (network_runner.py:125-153: the 29 rows ending at the last released
 *                       frame, zero rows before the first; deltas within the window).  conf = the model's decode; fired = the
 *                       model's TriggerDetector(2c bytes, cfg.sensitivity, cfg.trigger_level) over conf, in order
 *                       (runner.py:121-142); activations = fired count.  Equals one pb_update_ragged tick per chunk of a
 *                       fresh stream.  d_above and d_sum must be NULL.
 *   PB_CORPUS_SIMULATE  c = simulate's -c (samples between tests), c / hop_samples >= 1.  Windows end at frames
 *                       n_features + j (c / hop) < pb_mfcc_frames(L) (simulate.py:96-99's range).  fired =
 *                       TriggerDetector(c, sensitivity = threshold, trigger_level = 0) over raw (simulate.py:114-120,
 *                       refractory -(8 * 2048) // c); above = #(raw > threshold); sum = sum of raw in double (the reference
 *                       sums float32: the last bits differ).  Both comparisons are float32 against the threshold rounded to
 *                       float32, as numpy compares a float32 array with a Python float: raw > (float)(1 - threshold) and
 *                       raw > (float)threshold.  A recording with fewer than n_features + 1 frames yields 0 windows (the
 *                       reference's Runner.predict fails on its empty input). */
enum { PB_CORPUS_LISTENER = 0, PB_CORPUS_SIMULATE = 1 };

/* Windows one recording of n_samples yields under `schedule` (no device needed; cfg gives the front end), or a negative
 * pb_status: PB_ERR_INVALID for a null cfg, non-positive window / hop / n_features, a bad schedule or chunk, n_samples < 0. */
int64_t pb_corpus_windows(const pb_config* cfg, int32_t schedule, int64_t chunk, int64_t n_samples);

/* Scores n_rec recordings: recording r is d_pcm[h_offsets[r] .. h_offsets[r + 1]) (HOST offsets [n_rec + 1], non-decreasing,
 * any alignment; empty recordings yield 0 windows).  divisor: 32768 (buffer_to_audio, util.py:37) or 32767 (load_audio,
 * util.py:65), folded into the power scale as pb_mfcc folds 2^-15.  Window w of recording r is entry W_r + w, W_r the
 * exclusive prefix of pb_corpus_windows over the recordings.  Outputs are model-major over every bank model,
 * M = pb_num_models:
 *   d_raw [M][W_total] float32 (required), d_conf [M][W_total] float64, d_fired [M][W_total] uint8,
 *   d_activations, d_above [M][n_rec] int64, d_sum [M][n_rec] float64 -- all but d_raw optional (NULL).
 * Asynchronous on `stream`; h_offsets may be reused once the call returns.  The frames, window table and device offsets live
 * in a handle-owned workspace that grows on demand (about one row_stride-float row per hop of audio, 4 % of the int16
 * bytes at the defaults) and is freed by pb_destroy.  Two corpus calls on different CUDA streams are ordered by the library
 * (an event recorded after every call, failed ones included); the host waits for the previous call only when the workspace
 * must grow.
 * Profile slot 0 counts the MFCC kernels, slot 1 the network and trigger kernels.
 * At the aligned default geometry, recordings whose offset is a multiple of 8 samples (and d_pcm 16-byte aligned) take the
 * per-frame arithmetic of pb_mfcc's fast kernel, the others its generic kernel: frames are bit-identical to pb_mfcc of the
 * recording alone wherever both take the same kernel.
 * PB_ERR_INVALID: null handle, h_offsets or d_raw, a null d_pcm with samples, n_rec < 0, decreasing or negative offsets, a
 * bad divisor, schedule or chunk, d_above / d_sum with the listener schedule.  PB_ERR_STATE: slot 0 has no weights.
 * PB_ERR_CUDA: the workspace cannot be allocated (the handle is then unchanged). */
int pb_score_corpus(pb_handle* h, const int16_t* d_pcm, const int64_t* h_offsets, int64_t n_rec,
                    int32_t divisor, int32_t schedule, int64_t chunk, double threshold,
                    float* d_raw, double* d_conf, uint8_t* d_fired,
                    int64_t* d_activations, int64_t* d_above, double* d_sum, void* stream);
/* Pool models over recorded corpora: "how often does each custom wake word fire on this corpus" for many pool models in one
 * call.  Pool models h_model_ids[0 .. k) (HOST; repeats allowed, each gives its own identical row) score every window of the
 * n_rec recordings: a cross product.  Recordings, divisor, schedules, chunk and threshold mean exactly what they mean for
 * pb_score_corpus.  K1 and the window table run once per call, whatever k.
 *   - Outputs are model-major in the order of h_model_ids: d_raw, d_conf, d_fired [k][W_total]; d_activations, d_above,
 *     d_sum [k][n_rec].  Every output is optional, d_raw included, but not all of them at once.  Row i is bit-identical to
 *     the row pb_score_corpus writes for the same network in a bank of two or more models.
 *   - Listener schedule: each model's own decoder, cfg.sensitivity and cfg.trigger_level, refractory count from
 *     TriggerDetector(2c bytes), as pb_score_corpus.  Per-stream pool trigger settings do not apply (no stream is involved).
 *   - Reads and writes no stream state, pool assignments or pool detectors; needs no slot-0 weights; the bank is not scored.
 *   - Memory: the workspace of pb_score_corpus, shared with it, plus about 12 B per requested model.  Without d_raw, when a trigger pass is wanted, raw of a batch of max(1, 256 MB / (4 W_total)) rows is
 *     kept in the workspace (at most 256 MB, or one row's 4 W_total bytes): rows are scanned batch after batch, each followed by
 *     its trigger pass.
 *   - Asynchronous on `stream`, ordered against other corpus calls as pb_score_corpus.  pb_pool_load and pb_set_pool wait for
 *     queued calls, so a load after a call does not change what it scores.  Profile slot 0 counts K1, slot 1 the scans and
 *     trigger passes.  Every argument is checked before anything is enqueued, so a refused call changes no state.
 * PB_ERR_INVALID: pb_score_corpus's argument errors (but a null d_raw), every output null, k < 0, a null h_model_ids with
 * k > 0, an id outside [0, max_models) or a slot that holds no model.  PB_ERR_STATE: no pool.  PB_ERR_CUDA: the workspace
 * cannot be allocated (the handle is then unchanged). */
int pb_score_corpus_pool(pb_handle* h, const int16_t* d_pcm, const int64_t* h_offsets, int64_t n_rec,
                         const int32_t* h_model_ids, int64_t k,
                         int32_t divisor, int32_t schedule, int64_t chunk, double threshold,
                         float* d_raw, double* d_conf, uint8_t* d_fired,
                         int64_t* d_activations, int64_t* d_above, double* d_sum, void* stream);
/* Pool models over chosen recordings: each custom wake word over its owner's own audio (recorded samples, clips saved behind
 * past activations), and false-activation mining for pool models, without the cross product.  Pair p is pool slot
 * h_pair_models[p] over recording h_pair_recs[p] (both HOST, n_pairs entries; pairs may repeat and come in any order).
 * Recordings, divisor, schedules, chunk and threshold mean exactly what they mean for pb_score_corpus_pool, each model's own
 * decoder, sensitivity and trigger level included.  K1 runs over every recording, also one that no pair names.
 *   - Outputs are pair-major in request order.  d_raw, d_conf, d_fired [Wp]: pair p's windows are entries P[p] .. P[p+1] - 1,
 *     P the exclusive prefix over pairs of pb_corpus_windows of the pair's recording.  d_activations, d_above, d_sum
 *     [n_pairs].  Every output is optional (d_n_hits counts as one), but not all of them at once.  Pair p's outputs are
 *     bit-identical to the slice of recording h_pair_recs[p] in the row pb_score_corpus_pool writes for h_pair_models[p].
 *   - Hits (listener schedule only): with d_n_hits, *d_n_hits receives the number of pair-windows q in [0, Wp) whose decoded
 *     conf > hit_threshold (train_incremental.py:125's selection), and the first min(total, hit_capacity) of them go to
 *     d_hits [hit_capacity] (int64), in no particular order; the set is exact.  Hits need neither d_conf nor d_raw.
 *   - Pairs are scanned in batches of consecutive pairs of at most 2^25 pair-windows (a larger pair alone), each followed by
 *     its trigger and hit passes.  Scan tiles hold up to 64 consecutive pair-windows of one model, across the pairs of a run
 *     of consecutive pairs on that model: list a model's pairs together to fill them.
 *   - Memory: the workspace of pb_score_corpus, shared with it, plus 8 B per pair-window of the largest batch (its window
 *     table, at most 256 MB, or one pair's), 4 B more for raw when d_raw is NULL and a trigger or hit pass is wanted, and
 *     about 32 B per pair.
 *   - Reads and writes no stream state, pool assignments or pool detectors; needs no slot-0 weights.  Asynchronous on
 *     `stream`, ordered against other corpus calls as pb_score_corpus; pb_pool_load and pb_set_pool wait for queued calls.
 *     Profile slot 0 counts K1, slot 1 the scans, trigger and hit passes.  Every argument is checked before anything is
 *     enqueued, so a refused call changes no state.
 * PB_ERR_INVALID: pb_score_corpus_pool's argument errors, n_pairs outside [0, 2^31), a null pair array with n_pairs > 0, a
 * model id outside [0, max_models) or a slot that holds no model, a recording id outside [0, n_rec), hit_capacity < 0, a null
 * d_hits with hit_capacity > 0, d_hits without d_n_hits, hits with the simulate schedule.  PB_ERR_STATE: no pool.
 * PB_ERR_CUDA: the workspace cannot be allocated (the handle is then unchanged). */
int pb_score_corpus_pairs(pb_handle* h, const int16_t* d_pcm, const int64_t* h_offsets, int64_t n_rec,
                          const int32_t* h_pair_models, const int32_t* h_pair_recs, int64_t n_pairs,
                          int32_t divisor, int32_t schedule, int64_t chunk, double threshold,
                          float* d_raw, double* d_conf, uint8_t* d_fired,
                          int64_t* d_activations, int64_t* d_above, double* d_sum,
                          double hit_threshold, int64_t* d_hits, int64_t hit_capacity,
                          unsigned long long* d_n_hits, void* stream);
/* Pool models over labelled clips: one network input per recording, and per-model statistics over the outputs, for many
 * custom wake words in one call.  It is the device side of the reference's tools that work on Runner.predict(vectorize(clip)):
 * precise-test / precise-eval (precise/scripts/test.py, eval.py, precise/stats.py: true / false positives and negatives at a
 * threshold, the misclassified files), precise-graph (scripts/graph.py:147-152: the rates over ~100 thresholds) and
 * precise-calc-threshold (scripts/calc_threshold.py:66-83: mean and std of -log(1 / out - 1) over the positive clips).
 *   - Input per clip (vectorize, precise/vectorization.py:62-84): recording r, as pb_score_corpus takes recordings, cropped
 *     to its LAST max_samples samples (ListenerParams.max_samples) and framed from the cropped clip's first sample:
 *     nf = pb_mfcc_frames(min(L, max_samples)) frames, of which the network sees the last n_features, zero rows before them
 *     when there are fewer.  A clip too short for one frame scores the all-zero input.  No deltas (the pool's networks have
 *     none).  An empty recording is refused (the reference raises InvalidAudio).
 *   - Entries.  Cross product (h_pair_rows = h_pair_recs = NULL, n_pairs = 0): every model of h_model_ids [k] (HOST; pool
 *     slots, repeats allowed) over every recording; entry (i, r) at d_raw[i * n_rec + r].  Pairs (n_pairs > 0): entry p is
 *     model h_model_ids[h_pair_rows[p]] over recording h_pair_recs[p] (both HOST), at d_raw[p]: each word over its owner's
 *     own clips.  Scan tiles hold 64 consecutive pairs of one model: list a model's pairs together.  Raw outputs are
 *     bit-identical to pb_score_corpus_pool's / pb_score_corpus_pairs's for the same input rows.
 *   - Statistics, row i for h_model_ids[i] in both forms, all int64: exact, independent of the order of evaluation, and
 *     summed over calls by adding the arrays.  The label of an entry is h_targets[r] != 0 (HOST [n_rec]).  The call zeroes
 *     them first.
 *       d_count [k][2]               entries per label.
 *       d_hist  [k][2][2 n_thr + 1]  h_thresholds [n_thr] (HOST, 1 <= n_thr <= 1024) are rounded to float32 (numpy compares a
 *                                    float32 array with a Python float in float32) and must then be strictly ascending.  Bin
 *                                    2j + 1 counts raw == t_j, bin 2j counts t_(j-1) < raw < t_j (t_(-1) = -inf, t_n = +inf);
 *                                    NaN goes to bin 0.  Suffix sums give #(raw > t_j) (Stats.calc_metric, stats.py:102-107)
 *                                    and #(raw >= t_j) (Stats.num_correct, stats.py:54-56).
 *       d_fit   [k][2][3]            over entries with raw != 0 and raw != 1 (calc_threshold.py:66) and a finite
 *                                    v = -log((double)(1.0f / raw - 1.0f)) (the 1 / x - 1 in float32, as conf's decode; not
 *                                    finite for NaN and for float32 denormals): their number, the sum of llrint(v 2^32) and
 *                                    the sum of llrint(v^2 2^24).  |v| < 104, so no sum overflows while a (row, label) has at
 *                                    most 2^24 entries; a call with d_fit in which one would have more is refused.
 *     Misclassified entries (what precise-test lists): with d_n_miss, *d_n_miss receives the number of entries with
 *     (raw > (float)miss_threshold) != label, and the first min(total, miss_capacity) of them go to d_miss [miss_capacity] as
 *     i * n_rec + r (cross product) or p (pairs), in no particular order; the set is exact.
 *   - Every output is optional, d_raw included, but not all of them at once.  Without d_raw, raw of a batch (rows of at most
 *     256 MB, or 2^25 pairs) is kept in the corpus workspace, each batch followed by its statistics pass.
 *   - Reads and writes no stream state, pool assignment or detector; needs no slot-0 weights.  Asynchronous on `stream`,
 *     ordered against the corpus calls as pb_score_corpus (it shares their workspace).  Profile slot 0 counts K1, slot 1 the
 *     scans and statistics.  Every argument is checked before anything is enqueued, so a refused call changes no state.
 * PB_ERR_INVALID: pb_score_corpus's argument errors (but a null d_raw), every output null, max_samples < 1, a null h_targets,
 * an empty recording, k outside [0, 2^30), a null h_model_ids with k > 0, an id outside [0, max_models) or a slot that holds no
 * model, n_pairs outside [0, 2^31), one null pair array with n_pairs > 0, a row outside [0, k), a recording id outside
 * [0, n_rec), n_thr outside [0, 1024] or 0 with d_hist, null, NaN or not strictly ascending thresholds, miss_capacity < 0, a
 * null d_miss with miss_capacity > 0, d_miss without d_n_miss, more than 2^24 entries of one (row, label) with d_fit.
 * PB_ERR_STATE: no pool.  PB_ERR_CUDA: the workspace cannot be allocated (the handle is then unchanged). */
int pb_score_dataset(pb_handle* h, const int16_t* d_pcm, const int64_t* h_offsets, int64_t n_rec,
                     const uint8_t* h_targets, const int32_t* h_model_ids, int64_t k,
                     const int32_t* h_pair_rows, const int32_t* h_pair_recs, int64_t n_pairs,
                     int32_t divisor, int64_t max_samples, const double* h_thresholds, int32_t n_thr,
                     float* d_raw, int64_t* d_count, int64_t* d_hist, int64_t* d_fit,
                     double miss_threshold, int64_t* d_miss, int64_t miss_capacity, unsigned long long* d_n_miss,
                     void* stream);

/* ---- training (csrc/train.cuh): precise-train and precise-train-incremental's Keras fit (precise/model.py:57-91,
 * scripts/train.py:159-166, scripts/train_incremental.py:96-111) for many fused-family networks at once ---- */

/* The network input of each labelled clip, vectorize(clip) (precise/vectorization.py:62-84), as pb_score_dataset builds it:
 * recording r cropped to its last max_samples samples, the last n_features MFCC rows, zero rows in front when there are
 * fewer.  d_inputs [n_rec][n_features][feature_size] (DEVICE) receives rows bit-identical to the windows pb_score_dataset's
 * scans read.  Needs no pool.  Ordered against the corpus calls as pb_score_corpus (it shares their workspace).
 * PB_ERR_INVALID: pb_score_dataset's refusals of the clips (null or decreasing offsets, an empty recording, divisor,
 * max_samples < 1) and a null d_inputs.  PB_ERR_UNSUPPORTED: a front end outside the fused family (deltas, or feature size
 * > 16).  PB_ERR_CUDA: the workspace cannot be allocated. */
int pb_vectorize_clips(pb_handle* h, const int16_t* d_pcm, const int64_t* h_offsets, int64_t n_rec, int32_t divisor,
                       int64_t max_samples, float* d_inputs, void* stream);

/* Floats per network of pb_train's weight and accumulator arrays.  A row holds Keras's order, flat: kernel[F][3H],
 * recurrent[H][3H], bias[3H], dense_w[H], dense_b; the tail after 3H(F + H + 1) + H + 1 floats (2 977 at H = 24, F = 16) is
 * zero and stays zero. */
#define PB_TRAIN_STRIDE 2980

/* One trained network: hidden size (1 .. 24), PB_ACT_* and PB_RACT_* codes, and the seed of its shuffles and dropout masks. */
typedef struct pb_train_row {
    int32_t hidden;
    int32_t activation;
    int32_t recurrent_activation;
    uint32_t seed;
} pb_train_row;

/* Training settings (pb_train_opts_default: scripts/train.py's -e 10, -b 5000, -s 0.2 -> loss_bias 0.8 (train.py:86),
 * model.py:80's dropout 0.2, Keras RMSprop's lr 0.001, rho 0.9, epsilon 1e-7). */
typedef struct pb_train_opts {
    int32_t epochs;            /* >= 1                                                            */
    int32_t epoch0;            /* epoch number of the first epoch (>= 0): the shuffles and masks of a resumed fit */
    int32_t batch_size;        /* >= 1                                                            */
    float lr, rho, epsilon;    /* RMSprop: a = rho a + (1 - rho) g^2; w -= lr g / (sqrt(a) + epsilon) */
    float loss_bias;           /* [0, 1]: 1 - sensitivity                                          */
    float dropout;             /* [0, 1): input dropout rate                                      */
} pb_train_opts;

int pb_train_opts_default(pb_train_opts* opts);

/* Trains k networks on the handle's front end (feature size F, n_features steps T) over network inputs d_inputs
 * [n_rec][T][F] (DEVICE, pb_vectorize_clips') with labels h_targets [n_rec] (HOST, non-zero = wake word).
 *   - Entries as in pb_score_dataset: without pairs (n_pairs = 0) every row trains on every clip; with pairs, entry p belongs to
 *     row h_pair_rows[p] and uses clip h_pair_recs[p] (both HOST).  j, an entry's index within its row, counts in request order.
 *   - Per row and epoch e (epoch0 .. epoch0 + epochs - 1): the entries are sorted by (key(s, e, j, 0), j), cut into consecutive
 *     batches of batch_size (the last may be short) and each batch makes one RMSprop update of the mean loss over it:
 *     loss_bias mean(-(1-y) log(1-p+1e-7)) + (1-loss_bias) mean(-y log(p+1e-7)) (precise/functions.py:39-50), p the network's
 *     output with the entry's input dropout: feature f reaches gate g (z, r, h) scaled by 1.0f / (1.0f - dropout) iff
 *     float32((key(s, e, j, 1 + 3f + g) >> 40) 2^-24) >= dropout, else 0.  key(s, e, j, c) = mix(mix(mix(mix(s) + e) + j) + c) on
 *     uint64, mix the splitmix64 finalizer, s the row's seed.  Arithmetic is float32.
 *   - d_weights and d_rms [k][PB_TRAIN_STRIDE] (DEVICE) are read and updated in place: the optimizer's accumulators survive
 *     between calls, as the repeated fit of train_incremental keeps them.  d_loss [k][epochs] (DEVICE, optional) receives each
 *     epoch's loss, the batch-size-weighted mean of its batch losses (what Keras prints), as double.  A row with no entries is
 *     left untouched and its losses are NaN.
 *   - Results are bit-identical run to run, for a row alone or among any other rows in any order, and for E epochs in one call
 *     or in E calls with epoch0 advancing.
 *   - Asynchronous on `stream`, ordered against the corpus calls as pb_score_corpus.  Rows are trained in groups whose
 *     workspace stays under 256 MB.  Every argument is checked before anything is enqueued, so a refused call changes no buffer.
 * PB_ERR_INVALID: a null handle, opts, h_rows (k > 0), d_weights or d_rms (k > 0), d_inputs or h_targets (with entries), k
 * outside [0, 2^30), n_rec outside [0, 2^31), hidden outside [1, 24], an unknown activation code, n_pairs outside [0, 2^31), one
 * null pair array, a row outside [0, k), a clip outside [0, n_rec), epochs < 1, epoch0 < 0, batch_size < 1, a non-finite or
 * negative lr or epsilon, rho outside [0, 1), loss_bias outside [0, 1], dropout outside [0, 1).  PB_ERR_UNSUPPORTED: a front end
 * outside the fused family (deltas, or feature size > 16) or n_features > 112.  PB_ERR_CUDA: the workspace cannot be allocated. */
int pb_train(pb_handle* h, const float* d_inputs, int64_t n_rec, const uint8_t* h_targets, const pb_train_row* h_rows, int64_t k,
             const int32_t* h_pair_rows, const int32_t* h_pair_recs, int64_t n_pairs, const pb_train_opts* opts,
             float* d_weights, float* d_rms, double* d_loss, void* stream);

/* Each row's loss over all its entries as one batch, in request order, with the dropout masks of `epoch` (dropout 0: Keras's
 * evaluate, the val_loss train.py monitors), from d_weights (DEVICE, read only).  d_loss [k] (DEVICE) receives it (NaN for a
 * row with no entries); d_grad [k][PB_TRAIN_STRIDE] (DEVICE, optional) its gradient in the row layout (a row with no entries is
 * left untouched).  pb_train computes its updates with the same kernels.  Refusals as pb_train's, plus epoch < 0 and d_loss
 * and d_grad both null. */
int pb_train_loss(pb_handle* h, const float* d_inputs, int64_t n_rec, const uint8_t* h_targets, const pb_train_row* h_rows,
                  int64_t k, const int32_t* h_pair_rows, const int32_t* h_pair_recs, int64_t n_pairs, float loss_bias,
                  float dropout, int32_t epoch, const float* d_weights, double* d_loss, float* d_grad, void* stream);

/* Pinned host memory for pb_update_host / benchmarks. */
int pb_host_alloc(void** out, uint64_t bytes);
int pb_host_free(void* p);

/* Per-kernel device timing (CUDA events on the launching stream), for bench.py's roofline.
 * slot 0 = MFCC kernel, 1 = GRU(+decode+trigger) kernel (a bank tick or a corpus call: all its network kernels), 2 = decode-only kernel,
 * 3 = stream audio history kernels (the append of each tick, pb_read_history, switching and restarts; always 0 on a handle
 * without a history pool).
 * pb_profile_read synchronises the recorded events, returns accumulated ms and launch counts
 * since the last pb_profile_reset. */
int pb_profile_enable(pb_handle* h, int on);
int pb_profile_reset(pb_handle* h);
int pb_profile_read(pb_handle* h, double ms[4], uint64_t launches[4]);

/* Host copies of the device tables, for tests: mel filterbank [n_filt][n_fft/2+1] (float64),
 * decoder CDF (float64, length returned), and decoder range. */
int pb_get_filterbank(const pb_handle* h, double* h_out);
int64_t pb_get_cdf(const pb_handle* h, double* h_out, int64_t capacity, int32_t* min_out, int32_t* max_out);
/* Overrides the CDF table (same length as pb_get_cdf reports).  The Python host uploads the table
 * computed by numpy -- the library the reference builds it with (threshold_decoder.py:41,68-70) --
 * so decoded values are bit-identical to the reference's; the built-in table (libm exp) differs
 * from numpy's SIMD exp by at most an ulp per entry. */
int pb_set_cdf(pb_handle* h, const double* h_cd, int64_t len);

/* Test hook: route the aligned default geometry through the generic (any-alignment) MFCC kernels
 * instead of the warp-autonomous fast kernels, so both implementations are covered by parity tests. */
int pb_debug_force_generic(pb_handle* h, int on);
/* Test / A-B hook for the default network (H=20, F=13): 0 = automatic choice (warp-per-stream kernel up to 8192 streams per tick; above,
 * the fp16x3 mma.sync scan of csrc/gru_bank.cuh with one model), 1 = CUDA-core thread-per-stream kernel, 2 = the tensor-core scan
 * also for small batches.  Any other mode: PB_ERR_INVALID.  All variants are parity-tested (tests/test_gpu_parity.py). */
int pb_debug_gru_mode(pb_handle* h, int mode);
/* Test / A-B hook for the stateful tick's MFCC kernel (aligned default geometry).  0 = automatic: the pipelined FFT kernel on
 * the CUDA cores (csrc/mfcc_fast.cuh, mfcc_pipe_stream_kernel) where the geometry allows it, else the generic kernel; 2 = always
 * the FFT kernel it replaced (mfcc_fast_stream_kernel, bit-identical results); 3 = that kernel with its original 64-bit set-up; 4 / 5 / 6 = csrc/mfcc_mma.cuh, the DFT on mma.sync (stage 2 / both stages / both with a
 * shuffle epilogue; hop >= 512, chunk >= hop).  All variants are parity-tested (tests/test_gpu_parity.py). */
int pb_debug_k1_mode(pb_handle* h, int mode);
/* Test / A-B hook for the model pool's tiles: 0 = block tiles of 64 for each model's full groups, warp tiles of 16 for the
 * rest; 1 = warp tiles of 16 for every position.  Both score bit-identical outputs.  PB_ERR_STATE without a pool. */
int pb_debug_pool_tiles(pb_handle* h, int warp_only);
/* Test hook for pb_score_corpus_pool without d_raw: at most `rows` model rows per batch (rows >= 1), so that small corpora
 * reach the multi-batch path; 0 restores the default (the 256 MB raw cap).  PB_ERR_INVALID: null handle, rows < 0. */
int pb_debug_corpus_pool_rows(pb_handle* h, int64_t rows);
/* A/B hook for pb_score_corpus_pool's scan: nm models per CTA (1, 2, 4 or 8; 0 = the default), and grid order groups_fast
 * (1: consecutive CTAs take every model group of one window tile; 0: every tile of one group; -1 = the default).  Every
 * choice scores bit-identical outputs.  PB_ERR_INVALID: null handle, a value out of range. */
int pb_debug_corpus_pool_scan(pb_handle* h, int32_t nm, int32_t groups_fast);
/* Test hook for pb_score_corpus_pairs: at most `windows` pair-windows per batch (a larger pair still forms one batch), so that
 * small corpora reach the multi-batch path; 0 restores the default (2^25).  PB_ERR_INVALID: null handle, windows < 0. */
int pb_debug_corpus_pairs_batch(pb_handle* h, int64_t windows);
/* CPU model of a tensor-core formulation of the DFT (csrc/mfcc_tc.cuh: radix-16 butterflies, second stage as an fp16 hi / lo
 * matrix product) for one frame of 512 int16 samples -> |X[k]|^2, k = 0..256.  No device needed.  Test hook. */
int pb_debug_tc_dft_power(const int16_t* x512, double* power257);
/* CPU model of the k1 mode 4-6 kernel's DFT (csrc/mfcc_mma.cuh, its own tables) -> |X[k]|^2, k = 0..256.  Test hook. */
int pb_debug_mma_dft_power(const int16_t* x512, double* power257);
/* ... and of the whole MFCC for one frame (accumulators + mel / log / DCT epilogue with the tables of this configuration) -> out[min(n_filt, n_mfcc)].  No device needed.  Test hook. */
int pb_debug_tc_mfcc_frame(const pb_config* cfg, const int16_t* x512, float* out);
/* The same with both DFT stages as matrix products (csrc/mfcc_tc3.cuh: int16 split exactly into two fp16 pieces);
 * power257 (optional) receives |X[k]|^2 of the raw samples as the model's accumulators hold it.  No device needed.  Test hook. */
int pb_debug_tc3_mfcc_frame(const pb_config* cfg, const int16_t* x512, float* out, double* power257);

const char* pb_last_error(void);
int pb_abi_version(void);
const char* pb_build_info(void);

#ifdef __cplusplus
}
#endif
#endif /* PRECISE_B200_H */
