/* b200call.h -- C ABI of the b200call batched basecalling engine (libb200call.so).
 *
 * Drop-in boundary: dorado::basecall::ModelRunnerBase
 * (dorado/basecall/include/basecall/ModelRunnerBase.h:20-38).  The C++ adapter
 * include/B200ModelRunner.h implements that interface on top of the entry points below, replacing
 *   CudaModelRunner            dorado/basecall/CudaModelRunner.cpp:13-77
 *   CudaCaller                 dorado/basecall/CudaCaller.cpp:149-720
 *   CRFModel / TxModel (CUDA)  dorado/basecall/model/CRFModel.cpp:69-115, the run_koi paths under dorado/nn
 *   CUDADecoder                dorado/basecall/decode/CUDADecoder.cpp:17-173
 *   Koi                        cmake/Koi.cmake (closed libkoi.a)
 * No C++ types, exceptions or torch types cross this boundary: plain pointers and sizes only.
 * Every function returns B200_OK (0) or a negative b200_status; b200_last_error() gives the message
 * for the calling thread.  The library fails loudly (B200_ERR_CUDA) when no sm_90 (H100) device is usable;
 * there is no CPU fallback.
 */
#ifndef B200CALL_H
#define B200CALL_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_API __attribute__((visibility("default")))

typedef enum b200_status {
    B200_OK = 0,
    B200_ERR_INVALID = -1,     /* bad argument / unsupported model shape (std::invalid_argument in the adapter) */
    B200_ERR_CUDA = -2,        /* CUDA runtime / launch failure, no usable device */
    B200_ERR_UNSUPPORTED = -3, /* valid request outside what this build implements */
    B200_ERR_INTERNAL = -4
} b200_status;

/* config::Activation (dorado/config/include/config/common.h) */
enum { B200_ACT_SWISH = 0, B200_ACT_SWISH_CLAMP = 1, B200_ACT_TANH = 2 };
/* model family */
enum { B200_MODEL_LSTM = 0, B200_MODEL_TX = 1 };

/* config::ConvParams (dorado/config/include/config/common.h) */
typedef struct b200_conv_desc {
    int32_t insize, size, winlen, stride, activation;
} b200_conv_desc;

/* The fields of config::BasecallModelConfig that the hot path reads
 * (dorado/config/include/config/BasecallModelConfig.h). */
typedef struct b200_model_desc {
    int32_t model_type; /* B200_MODEL_LSTM | B200_MODEL_TX */
    int32_t num_convs;
    b200_conv_desc convs[8];
    int32_t state_len;
    int32_t outsize; /* 4^(state_len+1) */
    int32_t stride;  /* samples per output block */
    int32_t clamp;   /* config.clamp: scores clamped to +-5 (applied on decoder read) */
    float qscale, qbias;
    /* LSTM models (dorado/basecall/model/CRFModel.cpp:29-62) */
    int32_t lstm_size, lstm_layers;
    int32_t linear_bias;  /* config.bias */
    int32_t out_features; /* 0 = no linear decomposition */
    float crf_scale;      /* 5.0 => tanh(x)*5 on the last linear (pre-v4.x models) */
    /* transformer models (dorado/nn/TxModules.cpp, dorado/basecall/model/TxModel.cpp) */
    int32_t d_model, nhead, dim_feedforward, depth;
    int32_t attn_window_upper, attn_window_lower;
    int32_t upsample_scale, max_seq_len;
    float deepnorm_alpha, theta, tx_crf_scale;
    /* FLSTM models (config.lstm_inner_dim, BasecallModelConfig.h:145; dorado/nn/FLSTMStack.cpp): > 0 = every LSTM layer comes
     * as dn_weight_ih/hh [K, C], up_weight_ih/hh [4C, K], up_bias_ih/hh [4C]; the engine folds up x dn into the [4C, C] gate
     * matrices once at load time and runs the LSTM kernels unchanged. */
    int32_t lstm_inner_dim;
} b200_model_desc;

/* Host fp32 tensors, named and ordered as the reference's *.tensor files
 * (dorado/basecall/crf_utils.cpp:26-150); torch layouts ([out,in], conv [C_out,C_in,W]). */
typedef struct b200_tensor {
    const char* name;
    const float* data;
    int32_t ndim;
    int64_t dims[4];
} b200_tensor;

/* decode::DecoderOptions (dorado/basecall/include/basecall/DecodedChunk.h:15-23) */
typedef struct b200_decoder_options {
    int32_t beam_width; /* <= 32 */
    float beam_cut;
    float blank_score;
    float q_shift;
    float q_scale;
    float temperature; /* DecodedChunk.h:21; no decoder of the reference reads it (CPU, CUDA and Metal paths); kept so the
                          struct mirrors DecoderOptions field for field.  Must be 1. */
    int32_t move_pad;  /* DecodedChunk.h:22: never set in the reference tree and only forwarded to the closed Koi kernel
                          host_run_decode (CUDADecoder.cpp:100-104), so its meaning is not defined by any open source;
                          0 is accepted, anything else returns B200_ERR_UNSUPPORTED. */
} b200_decoder_options;

/* Result of one call_chunks(): pinned host arrays owned by the runner, rows of t_out bytes.
 * Chunk i of the batch: moves[i*t_out .. +t_out), sequence/qstring[i*t_out .. +n_bases[i]).
 * == decode::DecodedChunk {sequence, qstring, moves} (DecodedChunk.h:9-13). */
typedef struct b200_result {
    const uint8_t* moves;
    const char* sequence;
    const char* qstring;
    const int32_t* n_bases;
    int32_t t_out;
    int32_t num_chunks;
    const int32_t* n_moves; /* blocks of chunk i: moves[i*t_out .. +n_moves[i]); == t_out unless variable chunk sizes are in use */
} b200_result;

typedef struct b200_stats {
    int64_t batches_called;
    double model_decode_ms; /* GPU time forward+decode, CudaCaller.cpp:316-321 */
    double h2d_ms, d2h_ms;
    int64_t gpu_launches; /* kernels launched by this engine since creation */
    int64_t arena_bytes;
} b200_stats;

typedef struct b200_engine b200_engine; /* per-device model replica  (CudaCaller) */
typedef struct b200_runner b200_runner; /* per-thread batch slot set (CudaModelRunner) */

B200_API const char* b200_last_error(void);
B200_API const char* b200_version(void);
B200_API int b200_device_count(void);

B200_API void b200_default_decoder_options(b200_decoder_options* opts);

/* CudaCaller::CudaCaller (CudaCaller.cpp:149-202): upload + re-lay-out weights on `device`. */
B200_API int b200_engine_create(const b200_model_desc* desc,
                                const b200_tensor* tensors,
                                int32_t num_tensors,
                                int32_t device,
                                b200_engine** out);
B200_API int b200_engine_destroy(b200_engine* engine);
B200_API int b200_engine_get_stats(const b200_engine* engine, b200_stats* out);

/* CudaCaller lifecycle (CudaCaller.cpp:273-287): terminate refuses new batches and returns once the batches in flight have
 * finished; restart (idempotent, callable once per runner sharing the engine) admits batches again.  A call_chunks on a
 * terminated engine returns B200_ERR_INTERNAL ("terminated"). */
B200_API int b200_engine_terminate(b200_engine* engine);
B200_API int b200_engine_restart(b200_engine* engine);
/* Low-latency callers (PipelineType::simplex_low_latency, CudaCaller.cpp:126-138, 204-222): batch timeouts of 350 ms
 * instead of (300000, 30000), and runners created afterwards get highest-priority CUDA streams (the reference gives
 * low-latency callers a task queue of their own).  Call before creating runners. */
B200_API int b200_engine_set_low_latency(b200_engine* engine, int32_t on);
B200_API int32_t b200_engine_is_low_latency(const b200_engine* engine);
B200_API int b200_engine_batch_timeouts_ms(const b200_engine* engine, int32_t* first_chunk_ms, int32_t* last_chunk_ms);
/* num_runners of api::create_basecall_runners (api/runner_creation.cpp:46-130, default 2 per device): how many runners
 * (batches in flight) the caller is going to create on this engine.  Runners created afterwards size the grids of their
 * latency-bound kernels for that much concurrency (more chunks per CTA on fewer SMs, side by side with the other batches'
 * kernels).  Results do not depend on it.  Default 2. */
B200_API int b200_engine_set_num_runners(b200_engine* engine, int32_t num_runners);
B200_API int32_t b200_engine_num_runners(const b200_engine* engine);

/* CudaModelRunner::CudaModelRunner (CudaModelRunner.cpp:13-19) + CudaCaller::create_input/output_tensor
 * (CudaCaller.cpp:289-314): pinned fp16 input [batch, 1, chunk_size], pinned output, device arena. */
B200_API int b200_runner_create(b200_engine* engine, int32_t batch_size, int32_t chunk_size, b200_runner** out);
B200_API int b200_runner_destroy(b200_runner* runner);
B200_API int b200_runner_set_decoder_options(b200_runner* runner, const b200_decoder_options* opts);
B200_API int32_t b200_runner_batch_size(const b200_runner* runner);
B200_API int32_t b200_runner_chunk_size(const b200_runner* runner);
B200_API int32_t b200_runner_out_len(const b200_runner* runner); /* chunk_size / stride */

/* ModelRunnerBase::accept_chunk (CudaModelRunner.cpp:21-31): copy one chunk (fp16 bits, `len` samples,
 * len == chunk_size) into batch slot chunk_idx. */
B200_API int b200_runner_accept_chunk_f16(b200_runner* runner, int32_t chunk_idx, const uint16_t* samples, int64_t len);
/* Same, converting from fp32 on the way in (CPU ModelRunner's dtype, ModelRunner.cpp:47-49). */
B200_API int b200_runner_accept_chunk_f32(b200_runner* runner, int32_t chunk_idx, const float* samples, int64_t len);
/* Variable chunk sizes (SURVEY.md 8f row 1; CudaCaller::variable_chunk_sizes, api/runner_creation.cpp:24-42,
 * CudaModelRunner::accept_chunk CudaModelRunner.cpp:21-31, nn/AuxiliaryData.cpp:19-124, CUDADecoder.cpp:35-62,126-147):
 * chunks of different lengths share a batch, so a read's tail is not repeat-padded to chunk_size and the work for it shrinks.
 * b200_runner_variable_chunk_sizes() is 1 for the models the mode exists for (LSTM models with the cluster recurrence:
 * lstm_size 192 / 384); b200_runner_accept_chunk_var_f16 takes `len` samples, a positive multiple of the model stride and
 * <= chunk_size (BasecallerNode wraps a read's tail round to the next stride multiple, BasecallerNode.cpp:408-417).  The
 * reference packs the batch as one [1, C, sum T] row with an (offset, length) table; here every chunk keeps its slot and the
 * kernels read the length table: the convolutions see zero padding at the chunk's own end, the recurrence holds a zero
 * state outside 0 .. len-1 and a cluster only walks the steps one of its chunks is alive in, the decoder scans len/stride
 * blocks.  b200_result.n_moves gives the blocks of every row. */
B200_API int32_t b200_runner_variable_chunk_sizes(const b200_runner* runner);
B200_API int b200_runner_accept_chunk_var_f16(b200_runner* runner, int32_t chunk_idx, const uint16_t* samples, int64_t len);

/* Direct access to the pinned input (what the reference's accept_chunk writes through index_put_).  Slots keep their
 * content across calls; the call also turns every slot that holds a raw chunk back into an fp16 slot, so rows written
 * through the pointer are what the next call uploads (ask again after b200_runner_accept_raw_chunk). */
B200_API uint16_t* b200_runner_input(b200_runner* runner);

/* ModelRunnerBase::call_chunks (CudaCaller.cpp:224-271): H2D, forward, decode, D2H; blocking. */
B200_API int b200_runner_call_chunks(b200_runner* runner, int32_t num_chunks, b200_result* out);

/* Measurement hooks (bench.py): run `iters` forward+decode passes over the batch already resident on
 * the device (uploaded by the last call_chunks / upload) and report device time from CUDA events on the
 * runner's stream; decode_ms/forward_ms may be NULL. */
B200_API int b200_runner_upload(b200_runner* runner);
B200_API int b200_runner_step_device(b200_runner* runner, int32_t num_chunks, int32_t iters, float* total_ms,
                                     float* forward_ms, float* decode_ms);
/* The same with several runners of one engine in flight (the reference creates num_runners = 2 runners per device,
 * api/runner_creation.cpp:91-123): pass i runs on runners[i % n_runners], each on its own stream; total_ms is the
 * device time from the first launch to the last completion. */
B200_API int b200_runners_step_device(b200_runner** runners, int32_t n_runners, int32_t num_chunks, int32_t iters,
                                      float* total_ms);

/* ---- Front end of the path (SURVEY.md 8f rows 2-3): chunking, raw-signal scaling, stitching ------------------
 *
 * utils::generate_chunks (dorado/read_pipeline/base/chunk.cpp:11-47): chunk start offsets of a read of
 * `num_samples` samples.  Writes at most `capacity` offsets and always reports the full count.  The reference throws
 * on an empty read, stride 0, chunk_size 0 / not a multiple of stride / <= overlap, overlap not a multiple of stride:
 * those return B200_ERR_INVALID. */
B200_API int b200_generate_chunks(uint64_t num_samples,
                                  uint64_t chunk_size,
                                  uint64_t stride,
                                  uint64_t overlap,
                                  uint64_t* offsets,
                                  uint64_t capacity,
                                  uint64_t* count);

/* utils::generate_variable_chunks (dorado/read_pipeline/base/chunk.cpp:49-113), the chunking of the reference's
 * variable-chunk-size mode: near-equal chunks <= chunk_size whose interior boundaries lie on stride multiples.  Writes at
 * most `capacity` (first, second) pairs into intervals[2 * i], intervals[2 * i + 1] and always reports the full count.
 * Invalid arguments (those the reference throws on, incl. chunk_size == stride and overlap == 0 with stride != 1)
 * return B200_ERR_INVALID.  (The ragged batch layout that consumes these intervals is not implemented yet.) */
B200_API int b200_generate_variable_chunks(uint64_t num_samples,
                                           uint64_t chunk_size,
                                           uint64_t stride,
                                           uint64_t overlap,
                                           uint64_t* intervals,
                                           uint64_t capacity,
                                           uint64_t* count);

/* One chunk of a read given as RAW int16 signal: the device does what ScalerNode + BasecallerNode do on the host
 * in the reference --  x' = fp16((float(x) - shift) / scale)  (utils::shift_scale_tensor_i16_to_f16_inplace,
 * dorado/torch_utils/tensor_utils.cpp:100-143, called at read_pipeline/nodes/ScalerNode.cpp:226-229), the slice
 * raw[input_offset : input_offset + chunk_size] clamped at the read end, and repeat-padding of a short slice
 * (BasecallerNode.cpp:395-440) -- so int16 crosses PCIe once and no fp16 copy of the read is ever made on the host. */
typedef struct b200_raw_chunk {
    const int16_t* raw;    /* the read's whole raw signal (host memory) */
    uint64_t num_samples;  /* read length in samples */
    uint64_t input_offset; /* chunk start within the read (b200_generate_chunks) */
    float shift, scale;    /* ScalerNode's normalisation of this read */
} b200_raw_chunk;
/* accept_chunk for a raw chunk: stages the slice (only its un-padded samples) in pinned memory; the next
 * b200_runner_call_chunks uploads the staged int16 and runs the gather/scale kernel into the batch input.
 * Slots given through b200_runner_accept_chunk_f16/_f32 afterwards revert to the fp16 path. */
B200_API int b200_runner_accept_raw_chunk(b200_runner* runner, int32_t chunk_idx, const b200_raw_chunk* chunk);
/* Debug / test hook: run only the input stage (uploads + gather/scale kernel) for the first num_chunks slots and
 * copy the device-side fp16 batch input [num_chunks, chunk_size] back. */
B200_API int b200_runner_debug_read_input(b200_runner* runner, int32_t num_chunks, uint16_t* input_out);

/* utils::stitch_chunks (dorado/read_pipeline/base/stitch.cpp:12-96): merge the called chunks of one read, cutting
 * every overlap at its midpoint (in model-stride units), trimming a single short chunk to the read length and
 * dropping the partial-stride overhang.  `raw_samples` = ReadCommon::get_raw_data_samples(). */
typedef struct b200_called_chunk {
    uint64_t input_offset;   /* utils::Chunk::input_offset */
    uint64_t raw_chunk_size; /* utils::Chunk::raw_chunk_size */
    const uint8_t* moves;    /* n_moves = raw_chunk_size / stride entries */
    uint64_t n_moves;
    const char* sequence;    /* n_bases characters */
    const char* qstring;     /* n_bases characters */
    uint64_t n_bases;
} b200_called_chunk;
/* Output buffers must hold the sums of the inputs' n_moves / n_bases (upper bounds). */
B200_API int b200_stitch_chunks(const b200_called_chunk* chunks,
                                uint64_t n_chunks,
                                uint64_t raw_samples,
                                int32_t stride,
                                uint8_t* moves_out,
                                char* sequence_out,
                                char* qstring_out,
                                uint64_t* n_moves_out,
                                uint64_t* n_bases_out);

/* ---- Batch-size selection (SURVEY.md 8f row 4; CudaCaller::determine_batch_dims, CudaCaller.cpp:372-632) --------
 *
 * Device bytes one runner of (batch_size, chunk_size) allocates: exact, from the launch plan.  (The reference estimates
 * it from per-model tables of bytes per chunk-timestep, CudaCaller::calculate_memory_requirements, :323-370.) */
B200_API int b200_engine_runner_bytes(b200_engine* engine, int32_t batch_size, int32_t chunk_size, uint64_t* bytes);
/* The benchmark loop of determine_batch_dims (:530-557): for batch sizes granularity, 2*granularity, ... <=
 * max_batch_size, run the path twice on a scratch runner and keep the smaller time per chunk.  The reference times
 * the network forward only; here the decode runs on the device too, so forward + decode is timed.  Writes at most
 * `capacity` entries and reports the full count. */
B200_API int b200_engine_benchmark_batch_sizes(b200_engine* engine,
                                               int32_t chunk_size,
                                               int32_t granularity,
                                               int32_t max_batch_size,
                                               int32_t* batch_sizes,
                                               float* ms_per_chunk,
                                               int32_t capacity,
                                               int32_t* count);
/* CudaChunkBenchmarks::get_chunk_timings (dorado/basecall/benchmarks/CudaChunkBenchmarks.cpp:24-63): the pre-computed
 * timing table for (GPU name, model name), in ascending batch-size order; *count = 0 when there is none (the caller then
 * runs b200_engine_benchmark_batch_sizes, as CudaCaller.cpp:506-557 does).  b200_engine_gpu_name gives the name to look up. */
B200_API int b200_chunk_benchmarks_lookup(const char* gpu_name,
                                          const char* model_name,
                                          int32_t* batch_sizes,
                                          float* ms_per_chunk,
                                          int32_t capacity,
                                          int32_t* count);
B200_API int b200_engine_gpu_name(const b200_engine* engine, char* buf, uint64_t buf_len);

/* The selection rule of determine_batch_dims (:487-631) on such a table (ascending batch sizes): keep the entries that
 * improve on every smaller batch size, take the first of them within (1 + time_penalty) of the best time, and return
 * the largest kept batch size up to that entry that does not exceed max_batch_size (the memory cap); `granularity` if
 * none fits.  Pure host logic. */
B200_API int b200_select_batch_size(const int32_t* batch_sizes,
                                    const float* ms_per_chunk,
                                    int32_t count,
                                    int32_t max_batch_size,
                                    int32_t granularity,
                                    float time_penalty,
                                    int32_t* selected);

/* ---- Several devices in one process (SURVEY.md 8e) ---------------------------------------------------------------
 *
 * api::create_basecall_runners (dorado/api/runner_creation.cpp:46-130) creates one CudaCaller per device and num_runners
 * CudaModelRunners on each; BasecallerNode drives every runner from its own worker thread, all fed from shared chunk
 * queues (read_pipeline/nodes/BasecallerNode.cpp:300-352).  b200_pool_create is that: one engine per listed device,
 * runners_per_device runners each, one pinned host thread per runner (on the NUMA node of its device).
 * b200_pool_runner() hands out the runners for the adapter to wrap as ModelRunnerBase objects (runner_creation.cpp:115-123);
 * b200_pool_call_chunks is the worker loop itself for callers without a pipeline (bench, tests): `num_chunks` host chunks
 * (fp16 bits, [num_chunks][chunk_size]) are taken batch by batch from ONE shared cursor by whichever runner is free
 * (dynamic load balance; no collective, no inter-GPU traffic), results land in the caller's arrays with row pitch
 * b200_pool_out_len().  Blocking; returns the wall time in *seconds. */
typedef struct b200_pool b200_pool;
B200_API int b200_pool_create(const b200_model_desc* desc,
                              const b200_tensor* tensors,
                              int32_t num_tensors,
                              const int32_t* devices,
                              int32_t num_devices,
                              int32_t runners_per_device,
                              int32_t batch_size,
                              int32_t chunk_size,
                              b200_pool** out);
B200_API int b200_pool_destroy(b200_pool* pool);
B200_API int32_t b200_pool_num_runners(const b200_pool* pool);
B200_API b200_runner* b200_pool_runner(b200_pool* pool, int32_t index);
B200_API int32_t b200_pool_out_len(const b200_pool* pool);
/* per runner: host NUMA node its thread is pinned to (-1 = not pinned) and batches it has taken so far */
B200_API int b200_pool_runner_info(const b200_pool* pool, int32_t index, int32_t* numa_node, int64_t* batches);
B200_API int b200_pool_call_chunks(b200_pool* pool,
                                   const uint16_t* chunks,
                                   int64_t num_chunks,
                                   uint8_t* moves,
                                   char* sequence,
                                   char* qstring,
                                   int32_t* n_bases,
                                   double* seconds);

/* Stage-level entry points so scores and decode can be parity-checked independently (host buffers). */
B200_API int b200_runner_forward_scores(b200_runner* runner, int32_t num_chunks, uint16_t* scores_out /* [n,t_out,outsize] fp16 */);
B200_API int b200_decode_scores(int32_t device,
                                const uint16_t* scores /* [N,T,C] fp16 bits, host */,
                                int32_t N,
                                int32_t T,
                                int32_t C,
                                float clamp_val,
                                const b200_decoder_options* opts,
                                uint8_t* moves,
                                char* sequence,
                                char* qstring,
                                int32_t* n_bases);

/* One forward+decode pass with a CUDA event after every kernel launch.  Writes "name=ms;name=ms;..." (launch order,
 * device milliseconds) into buf. */
B200_API int b200_runner_profile(b200_runner* runner, int32_t num_chunks, char* buf, uint64_t buf_len);

/* Facts about the runner's launch plan as "key=value;...": the grid (CTAs) of kernels that are deliberately sized for a share
 * of the SMs so that several runners' kernels run side by side (b200_engine_set_num_runners), e.g.
 * "lstm_layer.ctas=32;lstm_layer.groups=2;lstm_layer.chunks_per_group=8".  Empty when every kernel spans the GPU. */
B200_API int b200_runner_plan_info(const b200_runner* runner, char* buf, uint64_t buf_len);

/* Debug: copy `bytes` of the runner's forward workspace (device) starting at `offset` to `dst` (host). */
B200_API int b200_runner_debug_read_workspace(b200_runner* runner, uint64_t offset, uint64_t bytes, void* dst);

/* Kernel-level test hooks (host buffers; used by tests/ only). */
B200_API int b200_test_gemm(int32_t device, const uint16_t* a /* [M,K] fp16 */, const uint16_t* b /* [N,K] fp16 */,
                            const float* bias /* [N] or NULL */, int32_t M, int32_t N, int32_t K, int32_t activation,
                            uint16_t* c /* [M,N] fp16 */);

#ifdef __cplusplus
}
#endif
#endif /* B200CALL_H */
