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
/* transformer precision (b200_model_desc.tx_precision) */
enum { B200_TX_FP16 = 0, B200_TX_FP8_FFN = 1, B200_TX_I8_QKV_FP8_FFN = 2 };
/* LSTM precision (b200_model_desc.lstm_precision) */
enum { B200_LSTM_FP16 = 0, B200_LSTM_INT8 = 1 };

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
    /* transformer models (dorado/nn/TxModules.cpp, dorado/basecall/model/TxModel.cpp).  Accepted shapes: d_model == 64 * nhead
     * (head dimension 64), d_model a multiple of 128 and at most 1536, dim_feedforward a multiple of 64, attention windows
     * 0 <= attn_window_upper, attn_window_lower <= 256 -- e.g. sup (512, 8 heads, (127, 128), 2048) and the 1536-wide
     * encoder (24 heads, (255, 256), 6144).  Anything else returns B200_ERR_UNSUPPORTED from b200_engine_create. */
    int32_t d_model, nhead, dim_feedforward, depth;
    int32_t attn_window_upper, attn_window_lower;
    int32_t upsample_scale, max_seq_len;
    float deepnorm_alpha, theta, tx_crf_scale;
    /* FLSTM models (config.lstm_inner_dim, BasecallModelConfig.h:145; dorado/nn/FLSTMStack.cpp): > 0 = every LSTM layer comes
     * as dn_weight_ih/hh [K, C], up_weight_ih/hh [4C, K], up_bias_ih/hh [4C]; the engine folds up x dn into the [4C, C] gate
     * matrices once at load time and runs the LSTM kernels unchanged. */
    int32_t lstm_inner_dim;
    /* Transformer precision.  B200_TX_FP16 (0, what a zero-initialised descriptor gets): every GEMM in fp16 with fp32
     * accumulation.  B200_TX_FP8_FFN (1): the reference's koi_use_f8 = 1, koi_use_i8 = 0 configuration
     * (dorado/nn/TxModules.cpp:477-479, 560-575, 596-697).  The weights are rounded to fp16 first; QKV, out_proj and both
     * RMSNorm gains then lose their low 4 mantissa bits (remove_bits = 4); fc1 and fc2 weights are cast to E4M3 without a
     * scale.  norm1 writes its output in fp16 and as an E4M3 copy, fc1 + SwiGLU reads the copy and writes E4M3, fc2 reads
     * that and writes fp16; both accumulate in fp32.  Shapes: those above, and dim_feedforward a multiple of 128 (fc2's K
     * in whole 128-byte E4M3 blocks; the engine does not pad it): others return B200_ERR_UNSUPPORTED.  On an LSTM model,
     * or any other value, b200_engine_create returns B200_ERR_INVALID.  b200_runner_plan_info reports "tx.fp8_ffn=1".
     * B200_TX_I8_QKV_FP8_FFN (2): koi_use_f8 = 1 with koi_use_i8 = 1, the reference's default on an H100
     * (TxModules.cpp:477-479, 936-961, 497-506, 611-616, 669, 713).  As B200_TX_FP8_FFN, and the fused QKV + RoPE projection
     * takes int8 operands: Wqkv is quantised per output row from the fp16 weights before remove_bits
     * (utils::quantize_tensor, evaluated in fp16), the encoder stack's input per token row by a device pass, and norm2 becomes
     * an explicit pass that writes the next layer's fp16 rows and their int8 copy; the s32 accumulator is converted to fp32
     * and multiplied by the row's and then the column's factor 1 / scale.  The same shapes and errors as B200_TX_FP8_FFN.
     * b200_runner_plan_info reports "tx.fp8_ffn=1;tx.int8_qkv=1". */
    int32_t tx_precision;
    /* LSTM precision.  B200_LSTM_FP16 (0, what a zero-initialised descriptor gets): fp16 operands, fp32 accumulation.
     * B200_LSTM_INT8 (1): the reference's CUTLASS_TNC_I8 layout (dorado/nn/ConvStack.cpp:66-74, LSTMStack.cpp:127-211,
     * CRFModules.cpp:103-117), its default for hac.  Per LSTM layer fp16(W_ih) | fp16(W_hh) are quantised to int8 as one
     * [4C, 2C] matrix with one fp16 scale per gate row (utils::quantize_tensor, evaluated in fp16 as the reference does); the
     * first CRF linear's weight likewise per output row.  The last convolution's tanh output and every h_t are stored as int8
     * round(127 v); the x-projection, the recurrence and that linear accumulate exactly in s32 and dequantise per row in fp32;
     * gx, the cell state and the scores keep their fp16 / fp32 types.  A second linear (out_features) stays fp16.  Shapes:
     * plain LSTM models with lstm_size 256 or 384 and a tanh last convolution; lstm_size 96 / 128 / 192 / 768 / 1024, another
     * last activation and FLSTM models return B200_ERR_UNSUPPORTED.  On a transformer model, or any other value,
     * b200_engine_create returns B200_ERR_INVALID.  b200_runner_plan_info reports "lstm.int8=1". */
    int32_t lstm_precision;
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
/* b200_model_desc grows by trailing fields, so the library has to know how much of it the caller's header declares:
 * b200_engine_create_sized reads desc_size bytes and takes every field beyond them as zero (a descriptor longer than the
 * library's own must be zero there, or B200_ERR_UNSUPPORTED).  b200_engine_create(desc, ...) in source compiled against
 * this header is b200_engine_create_sized(desc, sizeof(b200_model_desc), ...) (the macro below).  The exported symbol
 * b200_engine_create serves binaries built against earlier headers, which pass a shorter descriptor: it reads the fields
 * up to and including tx_precision, so such a binary keeps running in fp16 without being rebuilt.  The same holds for
 * b200_pool_create. */
B200_API int b200_engine_create_sized(const b200_model_desc* desc,
                                      size_t desc_size,
                                      const b200_tensor* tensors,
                                      int32_t num_tensors,
                                      int32_t device,
                                      b200_engine** out);
B200_API int b200_engine_create(const b200_model_desc* desc,
                                const b200_tensor* tensors,
                                int32_t num_tensors,
                                int32_t device,
                                b200_engine** out);
#define b200_engine_create(desc, tensors, num_tensors, device, out) \
    b200_engine_create_sized((desc), sizeof(b200_model_desc), (tensors), (num_tensors), (device), (out))
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
 * b200_runner_variable_chunk_sizes() is 1 for the models the mode exists for (plain LSTM models of lstm_size 128, 192, 256,
 * 384, 768 and 1024; not FLSTM).  The reference runs the mode only for multiples of 128 above 128
 * (check_variable_chunk_sizes_supported, api/runner_creation.cpp:28-31), so here 128 and 192 accept it where the reference
 * would call fixed-size chunks.  b200_runner_accept_chunk_var_f16 takes `len` samples, a positive multiple of the model stride and
 * <= chunk_size (BasecallerNode wraps a read's tail round to the next stride multiple, BasecallerNode.cpp:408-417).  The
 * reference packs the batch as one [1, C, sum T] row with an (offset, length) table; here every chunk keeps its slot and the
 * kernels read the length table: the convolutions see zero padding at the chunk's own end, the recurrence holds a zero
 * state outside 0 .. len-1 and a cluster (group of CTAs) only walks the steps one of its chunks is alive in, the decoder scans len/stride
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
 * it from per-model tables of bytes per chunk-timestep, CudaCaller::calculate_memory_requirements, :323-370.)  Returns
 * B200_ERR_INVALID for every shape b200_runner_create refuses. */
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
B200_API int b200_pool_create_sized(const b200_model_desc* desc,
                                    size_t desc_size,
                                    const b200_tensor* tensors,
                                    int32_t num_tensors,
                                    const int32_t* devices,
                                    int32_t num_devices,
                                    int32_t runners_per_device,
                                    int32_t batch_size,
                                    int32_t chunk_size,
                                    b200_pool** out);
/* As b200_engine_create: the symbol for binaries built against earlier headers, and the macro for this one. */
B200_API int b200_pool_create(const b200_model_desc* desc,
                              const b200_tensor* tensors,
                              int32_t num_tensors,
                              const int32_t* devices,
                              int32_t num_devices,
                              int32_t runners_per_device,
                              int32_t batch_size,
                              int32_t chunk_size,
                              b200_pool** out);
#define b200_pool_create(desc, tensors, num_tensors, devices, num_devices, runners_per_device, batch_size, chunk_size, out) \
    b200_pool_create_sized((desc), sizeof(b200_model_desc), (tensors), (num_tensors), (devices), (num_devices),          \
                           (runners_per_device), (batch_size), (chunk_size), (out))
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

/* Debug: copy `bytes` of the runner's forward workspace (device) starting at `offset` to `dst` (host).
 *
 * Transformer models: the workspace holds, in this order and each block starting on a 256-byte boundary,
 *   cbuf[0 .. num_convs - 2]   conv i's output, fp16 [N][t_i + 2 p_i + 16][size_i] with p_i = winlen_{i+1} / 2 zero rows
 *                              in front (conv i + 1 reads them as its padding), t_i the time length after conv i
 *   x, y, att                  fp16 [N * T][d_model] (T tokens per chunk)
 *   qkv                        fp16 [N * T][3 * d_model]
 *   hid                        fp16 [N * T][dim_feedforward]
 *   ups                        fp16 [N * T][upsample_scale * d_model]
 *   ss_a, ss_b                 fp32 [N * T][d_model / 32], partial sums of squares of the rows of x and of y
 * B200_DEBUG_TX_LAUNCHES=k, set before the runner is created, makes its forwards return after the first k kernel
 * launches of the plan (in the order b200_runner_profile lists them), so the buffers above can be read between any two
 * launches.  Unset, or k at least the plan's launch count, runs the whole plan. */
B200_API int b200_runner_debug_read_workspace(b200_runner* runner, uint64_t offset, uint64_t bytes, void* dst);

/* ---- Modified-base models (conv_lstm_v3) -----------------------------------------------------------------------
 *
 * Replaces ModBaseConvLSTMV3CUDAModel (dorado/modbase/nn/ModBaseModel.cpp:435-601) and the tensors of ModBaseRunner /
 * ModBaseCaller for one model.  The forward is ModBaseConvLSTMV3Model::forward (ModBaseModel.cpp:354-401):
 *   signal [1][sig_len] fp16 -> sig_convs[0..2];  k-mer one-hot [seq_len][kmer_len * 4] int8 -> seq_convs[0..1];
 *   concatenate along channels -> merge_conv -> LSTM forward in time -> LSTM reversed in time -> linear (+ bias)
 *   -> optional LinearUpsample -> softmax over num_out classes, returned as fp16 [out_len][num_out] per chunk.
 * Every convolution pads by winlen / 2 (ModsConv, ModBaseModel.cpp:91-97), so the encoders give
 * (len + 2 (winlen / 2) - winlen) / stride + 1 steps, e.g. 101 for 600 samples and the 6mA@v4 shapes. */
typedef struct b200_modbase_desc {
    b200_conv_desc sig_convs[3];   /* ModulesParams::signal_convs: 1 -> c1 (<= 16) -> 16 -> C_sig */
    b200_conv_desc seq_convs[2];   /* ModulesParams::sequence_convs: kmer_len * 4 -> 16 -> C_seq */
    b200_conv_desc merge_conv;     /* C_sig + C_seq -> lstm_size */
    int32_t lstm_size;             /* both LSTM layers: 128, 192, 256 or 384 (cluster kernel), 768 or 1024 (grid kernel) */
    int32_t num_out;               /* linear out_features */
    int32_t upsample_scale;        /* LinearUpsample scale_factor, 0 = no upsample */
    int32_t kmer_len;
    int32_t chunk_size;            /* ContextParams::chunk_size: signal samples per chunk */
} b200_modbase_desc;

/* Weights named as load_modbase_conv_lstm_weights reads them (ModBaseModel.cpp:49-75): "sig_conv1.weight.tensor", ...,
 * "lstm1.weight_ih_l0.tensor", ..., "fc.weight.tensor", "fc.bias.tensor", "linear_up.linear.weight.tensor", ... */
typedef struct b200_modbase_engine b200_modbase_engine;
typedef struct b200_modbase_runner b200_modbase_runner;

/* LSTM widths without a recurrence instantiation return B200_ERR_UNSUPPORTED. */
B200_API int b200_modbase_engine_create(const b200_modbase_desc* desc,
                                        const b200_tensor* tensors,
                                        int32_t num_tensors,
                                        int32_t device,
                                        b200_modbase_engine** out);
B200_API int b200_modbase_engine_destroy(b200_modbase_engine* engine);

/* Pinned input and output for batch_size chunks, device arena and launch plan; batch_size must be a multiple of 32
 * (B200_ERR_INVALID otherwise).  Runners of one engine run concurrently, each on its own stream. */
B200_API int b200_modbase_runner_create(b200_modbase_engine* engine, int32_t batch_size, b200_modbase_runner** out);
B200_API int b200_modbase_runner_destroy(b200_modbase_runner* runner);
B200_API int32_t b200_modbase_runner_batch_size(const b200_modbase_runner* runner);
B200_API int32_t b200_modbase_runner_sig_len(const b200_modbase_runner* runner); /* samples per chunk */
B200_API int32_t b200_modbase_runner_seq_len(const b200_modbase_runner* runner); /* k-mer steps per chunk */
B200_API int32_t b200_modbase_runner_out_len(const b200_modbase_runner* runner); /* output steps per chunk */
B200_API int32_t b200_modbase_runner_num_out(const b200_modbase_runner* runner);

/* ModBaseRunner::accept_chunk (dorado/modbase/ModBaseRunner.cpp:36-87): copy one chunk's signal (fp16 bits, sig_len
 * samples) and k-mer encoding (int8, seq_len * kmer_len * 4 values) into slot idx.  Any other length returns
 * B200_ERR_INVALID. */
B200_API int b200_modbase_runner_accept_chunk(b200_modbase_runner* runner,
                                              int32_t idx,
                                              const uint16_t* signal,
                                              int64_t sig_len,
                                              const int8_t* kmers,
                                              int64_t kmer_elems);
/* ModBaseRunner::call_chunks: H2D of the first num_chunks slots, forward, D2H; blocking.  *probs points at pinned fp16
 * [num_chunks][out_len * num_out] owned by the runner, valid until its next call. */
B200_API int b200_modbase_runner_call_chunks(b200_modbase_runner* runner, int32_t num_chunks, const uint16_t** probs);
/* One forward with a CUDA event after every kernel launch: "name=ms;name=ms;..." (launch order, device milliseconds). */
B200_API int b200_modbase_runner_profile(b200_modbase_runner* runner, char* buf, uint64_t buf_len);
/* Debug: copy `bytes` of the forward workspace starting at `offset` to dst.  The workspace starts with the LSTM
 * sequence buffer, fp16 [T][batch_size][lstm_size] (T = merge conv output steps): the merge conv output until the first
 * layer runs, then each layer's h.  B200_DEBUG_LSTM_LAYERS=k, set before the runner is created, stops its forwards
 * after k LSTM layers. */
B200_API int b200_modbase_runner_debug_read_workspace(b200_modbase_runner* runner, uint64_t offset, uint64_t bytes, void* dst);

/* Kernel-level test hooks (host buffers; used by tests/ only). */
/* The int8_qkv_fp8_ffn precision's device quantiser on fp16 rows [rows, cols] (cols a positive multiple of 128): int8 q
 * [rows, cols] and fp32 inv [rows] = 1 / float(fp16(128 / absmax)), bit for bit b200_test_quantize_rows' q and the reciprocal
 * of its scale (0 where the scale is +inf). */
B200_API int b200_test_quantize_act_rows(int32_t device, const uint16_t* f16, int32_t rows, int32_t cols, int8_t* q, float* inv);
/* Host only, no device: the int8_lstm weight quantisation of fp16 values [rows, cols], per row, as utils::quantize_tensor(w, 1)
 * computes it on an fp16 tensor: scale = fp16(128 / absmax), q = clip(round_half_even(fp16(w * scale)), -127, 127).  An all-zero
 * row gets q = 0 and scale = +inf (the engine dequantises such a row with the factor 0). */
B200_API int b200_test_quantize_rows(const uint16_t* f16, int32_t rows, int32_t cols, int8_t* q, uint16_t* scale);
/* Host only, no device: the fp8_ffn weight rounding.  to_e4m3: torch's float8_e4m3fn cast of each fp16 value (round to
 * nearest even; NaN beyond the range).  remove_bits: the reference's (bits + 2^(b-1)) & ~(2^b - 1) on the int16 view. */
B200_API int b200_test_to_e4m3(const uint16_t* f16, int64_t n, uint8_t* out);
B200_API int b200_test_remove_bits(const uint16_t* f16, int64_t n, int32_t bits, uint16_t* out);
/* The GEMM launched from every field the model plans set (dorado_b200/csrc/gemm.h, GemmDesc), on host buffers.  in_type
 * (A and W) and out_type are 0 fp16, 1 E4M3 or 2 int8 (GemmType); zero fields mean fp16.  Each buffer comes with its
 * length in elements of its type; a descriptor that would read or write beyond one, or that has no kernel form or sets an
 * input its form does not read (GemmDesc), returns B200_ERR_INVALID before anything is allocated.  Output offsets and
 * strides count elements of out_type.  Rows g = batch * rows_per_batch + r, r < rows_per_batch, read A at
 * batch * a_batch_stride + r * a_row_stride + k for k < (a_inner ? a_inner : K) (zeros beyond, up to K) and write
 * out + out_offset + (g / out_m1) * out_s0 + (g % out_m1) * out_s1 + n for n < N (N / 2 with SwiGLU).  The residual is
 * read at g * N + n, the partial sums of squares at g * parts + i.  out holds the caller's sentinel on entry and the
 * whole buffer on return.  out_ss, when not NULL, receives the N / 32 partials of every row (NaN where none was written).
 * act 5 (RoPE) takes the model's own table for theta and max_seq_len, and rotates position g % rope_T. */
typedef struct b200_gemm_test_desc {
    const void* a;             int64_t a_len;         /* in_type, flat: overlapping and padded views are the caller's */
    const void* w;             int64_t w_len;         /* in_type [N][K] */
    const float* bias;         int64_t bias_len;      /* [N] or NULL */
    const uint16_t* residual;  int64_t residual_len;  /* fp16 or NULL */
    const float* res_gain;     int64_t res_gain_len;  /* [N] or NULL */
    const float* a_ss;         int64_t a_ss_len;      /* [rows][a_ss_parts] or NULL */
    const float* res_ss;       int64_t res_ss_len;    /* [rows][res_ss_parts] or NULL */
    void* out;                 int64_t out_len;       /* out_type */
    float* out_ss;             int64_t out_ss_len;    /* [rows][N / 32] or NULL */
    int32_t batches, rows_per_batch;
    int64_t a_row_stride, a_batch_stride;
    int32_t a_inner, K, N, act;
    int64_t out_offset, out_m1, out_s0, out_s1;
    float alpha;
    int32_t a_ss_parts, res_ss_parts, norm_dim;
    float norm_eps;
    int32_t max_ctas;
    float theta;
    int32_t max_seq_len, rope_T, rope_cols;
    int32_t in_type, out_type;
    const float* col_scale;    int64_t col_scale_len; /* [N] or NULL: required with int8 operands */
    const float* row_scale;    int64_t row_scale_len; /* [rows] or NULL: int8 operands with per-row factors */
} b200_gemm_test_desc;
B200_API int b200_test_gemm_desc(int32_t device, const b200_gemm_test_desc* desc);
/* The transformer's sliding-window attention kernel, launched exactly as the model launches it: qkv of N chunks of T tokens
 * (q and k already rotated), query i of a chunk attends keys j with -win_upper <= j - i <= win_lower, softmax scale 1/8.
 * Windows outside [0, 256] return B200_ERR_UNSUPPORTED. */
B200_API int b200_test_attention(int32_t device, const uint16_t* qkv /* [N*T][3][H][64] fp16 */, int32_t N, int32_t T,
                                 int32_t H, int32_t win_upper, int32_t win_lower, uint16_t* out /* [N*T][H*64] fp16 */);

#ifdef __cplusplus
}
#endif
#endif /* B200CALL_H */
