// C ABI of libb200call.so (declared in include/b200call.h): status codes instead of exceptions,
// plain pointers and sizes, no torch types.
#include "b200call.h"

#include "common.cuh"
#include "decode.h"
#include "engine.h"

#include <cmath>
#include <cstring>
#include <limits>
#include <string>

namespace {

thread_local std::string g_last_error;

template <typename F>
int guarded(F&& fn) {
    try {
        fn();
        return B200_OK;
    } catch (const std::invalid_argument& e) {
        g_last_error = e.what();
        return B200_ERR_INVALID;
    } catch (const b200::CudaError& e) {
        g_last_error = e.what();
        return B200_ERR_CUDA;
    } catch (const b200::Unsupported& e) {
        g_last_error = e.what();
        return B200_ERR_UNSUPPORTED;
    } catch (const std::exception& e) {
        g_last_error = e.what();
        return B200_ERR_INTERNAL;
    }
}

}  // namespace

extern "C" {

const char* b200_last_error(void) { return g_last_error.c_str(); }
const char* b200_version(void) { return "b200call 0.1 (sm_90a)"; }

int b200_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

void b200_default_decoder_options(b200_decoder_options* o) {
    // decode::DecoderOptions defaults (dorado/basecall/include/basecall/DecodedChunk.h:15-23)
    o->beam_width = 32;
    o->beam_cut = 100.0f;
    o->blank_score = 2.0f;
    o->q_shift = 0.0f;
    o->q_scale = 1.0f;
    o->temperature = 1.0f;
    o->move_pad = 0;
}

int b200_engine_create(const b200_model_desc* desc, const b200_tensor* tensors, int32_t num_tensors, int32_t device,
                       b200_engine** out) {
    return guarded([&] {
        if (!desc || !tensors || !out) throw std::invalid_argument("b200_engine_create: null argument");
        *out = reinterpret_cast<b200_engine*>(new b200::Engine(*desc, tensors, num_tensors, device));
    });
}

int b200_engine_destroy(b200_engine* e) {
    return guarded([&] { delete reinterpret_cast<b200::Engine*>(e); });
}

int b200_engine_get_stats(const b200_engine* e, b200_stats* out) {
    return guarded([&] {
        if (!e || !out) throw std::invalid_argument("b200_engine_get_stats: null argument");
        *out = reinterpret_cast<const b200::Engine*>(e)->stats();
    });
}

int b200_chunk_benchmarks_lookup(const char* gpu_name, const char* model_name, int32_t* batch_sizes, float* ms_per_chunk,
                                 int32_t capacity, int32_t* count) {
    return guarded([&] {
        const int n = b200::lookup_chunk_benchmarks(gpu_name, model_name, batch_sizes, ms_per_chunk, capacity);
        if (count) *count = n;
    });
}

int b200_engine_gpu_name(const b200_engine* e, char* buf, uint64_t buf_len) {
    return guarded([&] {
        if (!e || !buf || buf_len == 0) throw std::invalid_argument("b200_engine_gpu_name: null argument");
        const std::string n = b200::device_name(reinterpret_cast<const b200::Engine*>(e)->device());
        std::strncpy(buf, n.c_str(), buf_len - 1);
        buf[buf_len - 1] = '\0';
    });
}

int b200_engine_terminate(b200_engine* e) {
    return guarded([&] {
        if (!e) throw std::invalid_argument("b200_engine_terminate: null argument");
        reinterpret_cast<b200::Engine*>(e)->terminate();
    });
}

int b200_engine_restart(b200_engine* e) {
    return guarded([&] {
        if (!e) throw std::invalid_argument("b200_engine_restart: null argument");
        reinterpret_cast<b200::Engine*>(e)->restart();
    });
}

int b200_engine_set_low_latency(b200_engine* e, int32_t on) {
    return guarded([&] {
        if (!e) throw std::invalid_argument("b200_engine_set_low_latency: null argument");
        reinterpret_cast<b200::Engine*>(e)->set_low_latency(on != 0);
    });
}

int b200_engine_set_num_runners(b200_engine* e, int32_t num_runners) {
    return guarded([&] {
        if (!e || num_runners < 1) throw std::invalid_argument("b200_engine_set_num_runners: null engine or num_runners < 1");
        reinterpret_cast<b200::Engine*>(e)->set_num_runners(num_runners);
    });
}

int32_t b200_engine_num_runners(const b200_engine* e) { return e ? reinterpret_cast<const b200::Engine*>(e)->num_runners() : 0; }

int32_t b200_engine_is_low_latency(const b200_engine* e) { return e && reinterpret_cast<const b200::Engine*>(e)->low_latency(); }

int b200_engine_batch_timeouts_ms(const b200_engine* e, int32_t* first_chunk_ms, int32_t* last_chunk_ms) {
    return guarded([&] {
        if (!e) throw std::invalid_argument("b200_engine_batch_timeouts_ms: null argument");
        int a = 0, b = 0;
        reinterpret_cast<const b200::Engine*>(e)->batch_timeouts_ms(&a, &b);
        if (first_chunk_ms) *first_chunk_ms = a;
        if (last_chunk_ms) *last_chunk_ms = b;
    });
}

int b200_pool_create(const b200_model_desc* desc, const b200_tensor* tensors, int32_t num_tensors, const int32_t* devices,
                     int32_t num_devices, int32_t runners_per_device, int32_t batch_size, int32_t chunk_size, b200_pool** out) {
    return guarded([&] {
        if (!desc || !tensors || !devices || !out) throw std::invalid_argument("b200_pool_create: null argument");
        *out = reinterpret_cast<b200_pool*>(
                new b200::Pool(*desc, tensors, num_tensors, devices, num_devices, runners_per_device, batch_size, chunk_size));
    });
}

int b200_pool_destroy(b200_pool* p) {
    return guarded([&] { delete reinterpret_cast<b200::Pool*>(p); });
}

int32_t b200_pool_num_runners(const b200_pool* p) { return p ? reinterpret_cast<const b200::Pool*>(p)->num_runners() : 0; }
int32_t b200_pool_out_len(const b200_pool* p) { return p ? reinterpret_cast<const b200::Pool*>(p)->out_len() : 0; }

b200_runner* b200_pool_runner(b200_pool* p, int32_t index) {
    return p ? reinterpret_cast<b200_runner*>(reinterpret_cast<b200::Pool*>(p)->runner(index)) : nullptr;
}

int b200_pool_runner_info(const b200_pool* p, int32_t index, int32_t* numa_node, int64_t* batches) {
    return guarded([&] {
        if (!p) throw std::invalid_argument("b200_pool_runner_info: null argument");
        const auto* pool = reinterpret_cast<const b200::Pool*>(p);
        if (index < 0 || index >= pool->num_runners()) throw std::invalid_argument("b200_pool_runner_info: index out of range");
        if (numa_node) *numa_node = pool->runner_numa_node(index);
        if (batches) *batches = pool->runner_batches(index);
    });
}

int b200_pool_call_chunks(b200_pool* p, const uint16_t* chunks, int64_t num_chunks, uint8_t* moves, char* sequence,
                          char* qstring, int32_t* n_bases, double* seconds) {
    return guarded([&] {
        if (!p) throw std::invalid_argument("b200_pool_call_chunks: null argument");
        const double s = reinterpret_cast<b200::Pool*>(p)->call_chunks(chunks, num_chunks, moves, sequence, qstring, n_bases);
        if (seconds) *seconds = s;
    });
}

int b200_runner_create(b200_engine* e, int32_t batch_size, int32_t chunk_size, b200_runner** out) {
    return guarded([&] {
        if (!e || !out) throw std::invalid_argument("b200_runner_create: null argument");
        *out = reinterpret_cast<b200_runner*>(new b200::Runner(*reinterpret_cast<b200::Engine*>(e), batch_size, chunk_size));
    });
}

int b200_runner_destroy(b200_runner* r) {
    return guarded([&] { delete reinterpret_cast<b200::Runner*>(r); });
}

int b200_runner_set_decoder_options(b200_runner* r, const b200_decoder_options* o) {
    return guarded([&] {
        if (!r || !o) throw std::invalid_argument("b200_runner_set_decoder_options: null argument");
        reinterpret_cast<b200::Runner*>(r)->set_decoder_options(*o);
    });
}

int32_t b200_runner_batch_size(const b200_runner* r) { return r ? reinterpret_cast<const b200::Runner*>(r)->batch_size() : 0; }
int32_t b200_runner_chunk_size(const b200_runner* r) { return r ? reinterpret_cast<const b200::Runner*>(r)->chunk_size() : 0; }
int32_t b200_runner_out_len(const b200_runner* r) { return r ? reinterpret_cast<const b200::Runner*>(r)->out_len() : 0; }

int b200_runner_accept_chunk_f16(b200_runner* r, int32_t idx, const uint16_t* samples, int64_t len) {
    return guarded([&] {
        if (!r || !samples) throw std::invalid_argument("b200_runner_accept_chunk_f16: null argument");
        reinterpret_cast<b200::Runner*>(r)->accept_chunk_f16(idx, samples, len);
    });
}

int b200_runner_accept_chunk_f32(b200_runner* r, int32_t idx, const float* samples, int64_t len) {
    return guarded([&] {
        if (!r || !samples) throw std::invalid_argument("b200_runner_accept_chunk_f32: null argument");
        reinterpret_cast<b200::Runner*>(r)->accept_chunk_f32(idx, samples, len);
    });
}

int32_t b200_runner_variable_chunk_sizes(const b200_runner* r) {
    return r && reinterpret_cast<const b200::Runner*>(r)->variable_chunk_sizes();
}

int b200_runner_accept_chunk_var_f16(b200_runner* r, int32_t idx, const uint16_t* samples, int64_t len) {
    return guarded([&] {
        if (!r || !samples) throw std::invalid_argument("b200_runner_accept_chunk_var_f16: null argument");
        reinterpret_cast<b200::Runner*>(r)->accept_chunk_var_f16(idx, samples, len);
    });
}

uint16_t* b200_runner_input(b200_runner* r) { return r ? reinterpret_cast<b200::Runner*>(r)->input() : nullptr; }

int b200_runner_call_chunks(b200_runner* r, int32_t num_chunks, b200_result* out) {
    return guarded([&] {
        if (!r || !out) throw std::invalid_argument("b200_runner_call_chunks: null argument");
        *out = reinterpret_cast<b200::Runner*>(r)->call_chunks(num_chunks);
    });
}

int b200_generate_chunks(uint64_t num_samples, uint64_t chunk_size, uint64_t stride, uint64_t overlap, uint64_t* offsets,
                         uint64_t capacity, uint64_t* count) {
    return guarded([&] {
        if (!count || (!offsets && capacity)) throw std::invalid_argument("b200_generate_chunks: null argument");
        *count = b200::generate_chunks(num_samples, chunk_size, stride, overlap, offsets, capacity);
    });
}

int b200_generate_variable_chunks(uint64_t num_samples, uint64_t chunk_size, uint64_t stride, uint64_t overlap,
                                  uint64_t* intervals, uint64_t capacity, uint64_t* count) {
    return guarded([&] {
        if (!count || (!intervals && capacity)) throw std::invalid_argument("b200_generate_variable_chunks: null argument");
        *count = b200::generate_variable_chunks(num_samples, chunk_size, stride, overlap, intervals, capacity);
    });
}

int b200_stitch_chunks(const b200_called_chunk* chunks, uint64_t n_chunks, uint64_t raw_samples, int32_t stride,
                       uint8_t* moves_out, char* sequence_out, char* qstring_out, uint64_t* n_moves_out,
                       uint64_t* n_bases_out) {
    return guarded([&] {
        if (!moves_out || !sequence_out || !qstring_out || !n_moves_out || !n_bases_out) {
            throw std::invalid_argument("b200_stitch_chunks: null argument");
        }
        b200::stitch_chunks(chunks, n_chunks, raw_samples, stride, moves_out, sequence_out, qstring_out, n_moves_out,
                            n_bases_out);
    });
}

int b200_runner_accept_raw_chunk(b200_runner* r, int32_t chunk_idx, const b200_raw_chunk* chunk) {
    return guarded([&] {
        if (!r || !chunk) throw std::invalid_argument("b200_runner_accept_raw_chunk: null argument");
        reinterpret_cast<b200::Runner*>(r)->accept_raw_chunk(chunk_idx, *chunk);
    });
}

int b200_runner_debug_read_input(b200_runner* r, int32_t num_chunks, uint16_t* input_out) {
    return guarded([&] {
        if (!r) throw std::invalid_argument("b200_runner_debug_read_input: null argument");
        reinterpret_cast<b200::Runner*>(r)->debug_read_input(num_chunks, input_out);
    });
}

int b200_engine_runner_bytes(b200_engine* e, int32_t batch_size, int32_t chunk_size, uint64_t* bytes) {
    return guarded([&] {
        if (!e || !bytes) throw std::invalid_argument("b200_engine_runner_bytes: null argument");
        *bytes = b200::runner_device_bytes(*reinterpret_cast<b200::Engine*>(e), batch_size, chunk_size);
    });
}

int b200_engine_benchmark_batch_sizes(b200_engine* e, int32_t chunk_size, int32_t granularity, int32_t max_batch_size,
                                      int32_t* batch_sizes, float* ms_per_chunk, int32_t capacity, int32_t* count) {
    return guarded([&] {
        if (!e || !count || capacity < 0) throw std::invalid_argument("b200_engine_benchmark_batch_sizes: bad argument");
        *count = b200::benchmark_batch_sizes(*reinterpret_cast<b200::Engine*>(e), chunk_size, granularity, max_batch_size,
                                             batch_sizes, ms_per_chunk, capacity);
    });
}

int b200_select_batch_size(const int32_t* batch_sizes, const float* ms_per_chunk, int32_t count, int32_t max_batch_size,
                           int32_t granularity, float time_penalty, int32_t* selected) {
    return guarded([&] {
        if (!selected) throw std::invalid_argument("b200_select_batch_size: null argument");
        *selected = b200::select_batch_size(batch_sizes, ms_per_chunk, count, max_batch_size, granularity, time_penalty);
    });
}

int b200_runner_upload(b200_runner* r) {
    return guarded([&] {
        if (!r) throw std::invalid_argument("b200_runner_upload: null argument");
        reinterpret_cast<b200::Runner*>(r)->upload();
    });
}

int b200_runners_step_device(b200_runner** runners, int32_t n_runners, int32_t num_chunks, int32_t iters, float* total_ms) {
    return guarded([&] {
        if (!runners || !total_ms) throw std::invalid_argument("b200_runners_step_device: null argument");
        b200::pipelined_steps(reinterpret_cast<b200::Runner**>(runners), n_runners, num_chunks, iters, total_ms);
    });
}

int b200_runner_step_device(b200_runner* r, int32_t num_chunks, int32_t iters, float* total_ms, float* forward_ms,
                            float* decode_ms) {
    return guarded([&] {
        if (!r || !total_ms) throw std::invalid_argument("b200_runner_step_device: null argument");
        reinterpret_cast<b200::Runner*>(r)->step_device(num_chunks, iters, total_ms, forward_ms, decode_ms);
    });
}

int b200_runner_forward_scores(b200_runner* r, int32_t num_chunks, uint16_t* scores_out) {
    return guarded([&] {
        if (!r || !scores_out) throw std::invalid_argument("b200_runner_forward_scores: null argument");
        reinterpret_cast<b200::Runner*>(r)->forward_scores_to_host(num_chunks, scores_out);
    });
}

int b200_runner_profile(b200_runner* r, int32_t num_chunks, char* buf, uint64_t buf_len) {
    return guarded([&] {
        if (!r || !buf || buf_len == 0) throw std::invalid_argument("b200_runner_profile: null argument");
        const std::string s = reinterpret_cast<b200::Runner*>(r)->profile(num_chunks);
        std::strncpy(buf, s.c_str(), buf_len - 1);
        buf[buf_len - 1] = 0;
    });
}

int b200_runner_plan_info(const b200_runner* r, char* buf, uint64_t buf_len) {
    return guarded([&] {
        if (!r || !buf || buf_len == 0) throw std::invalid_argument("b200_runner_plan_info: null argument");
        const std::string s = reinterpret_cast<const b200::Runner*>(r)->plan_info();
        std::strncpy(buf, s.c_str(), buf_len - 1);
        buf[buf_len - 1] = 0;
    });
}

int b200_runner_debug_read_workspace(b200_runner* r, uint64_t offset, uint64_t bytes, void* dst) {
    return guarded([&] {
        if (!r || !dst) throw std::invalid_argument("debug_read_workspace: null argument");
        reinterpret_cast<b200::Runner*>(r)->debug_read_workspace(offset, bytes, dst);
    });
}

int b200_decode_scores(int32_t device, const uint16_t* scores, int32_t N, int32_t T, int32_t C, float clamp_val,
                       const b200_decoder_options* opts, uint8_t* moves, char* sequence, char* qstring,
                       int32_t* n_bases) {
    return guarded([&] {
        if (!scores || !opts || !moves || !sequence || !qstring || !n_bases) {
            throw std::invalid_argument("b200_decode_scores: null argument");
        }
        b200::decode_host_scores(device, scores, N, T, C, clamp_val, *opts, moves, sequence, qstring, n_bases);
    });
}

int b200_test_gemm(int32_t device, const uint16_t* a, const uint16_t* b, const float* bias, int32_t M, int32_t N,
                   int32_t K, int32_t activation, uint16_t* c) {
    return guarded([&] {
        if (!a || !b || !c) throw std::invalid_argument("b200_test_gemm: null argument");
        b200::test_gemm_host(device, a, b, bias, M, N, K, activation, c);
    });
}

}  // extern "C"
