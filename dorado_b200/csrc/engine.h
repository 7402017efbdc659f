// Host side of libb200call.so: Engine (one model replica per device, the reference's CudaCaller) and
// Runner (pinned batch slots + device arena, the reference's CudaModelRunner).
#pragma once

#include "b200call.h"
#include "b200_crf_math.h"
#include "frontend.h"
#include "common.cuh"

#include <atomic>
#include <condition_variable>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>

namespace b200 {

struct Unsupported : std::runtime_error {
    using std::runtime_error::runtime_error;
};

// Simple bump arena over one cudaMalloc (the reference plans its working memory the same way:
// dorado/nn/WorkingMemory.cpp:27-112). 256-byte aligned slices.
class Arena {
public:
    Arena() = default;
    ~Arena();
    Arena(const Arena&) = delete;
    Arena& operator=(const Arena&) = delete;
    void reserve(size_t bytes);
    void* take(size_t bytes);
    void reset() { m_off = 0; }
    size_t capacity() const { return m_cap; }

private:
    unsigned char* m_base = nullptr;
    size_t m_cap = 0, m_off = 0;
};

// Network forward for one fixed batch shape: fp16 signal [N][T_in] on device -> fp16 scores
// [N][T_out][outsize] on device.  A plan owns its tensor maps and launch parameters (all pointers are
// fixed slices of the runner's arena), so a forward is just a sequence of launches.  The whole batch
// is always computed (slots beyond num_chunks hold stale data and are ignored, as in the reference).
// Optional per-kernel timing: mark() records an event after each launch; report() turns them into
// (kernel name, milliseconds) pairs once the stream has drained.  Used by bench.py for the roofline line.
struct ProfileSink {
    std::vector<cudaEvent_t> events;
    std::vector<std::string> names;
    void begin(cudaStream_t s);
    void mark(const char* name, cudaStream_t s);
    std::vector<std::pair<std::string, float>> report();
    ~ProfileSink();
};

class ForwardPlan {
public:
    virtual ~ForwardPlan() = default;
    virtual void run(cudaStream_t stream, ProfileSink* prof = nullptr) = 0;
    virtual int launches() const = 0;
    // Variable chunk sizes: device array of per-chunk lengths in samples (multiples of the stride, <= T_in), read by the
    // kernels at run time.  Plans of models without that mode ignore it.
    virtual void set_chunk_lengths(const int32_t* /*d_lens*/) {}
    // "key=value;..." facts about the launch plan that measurements need (grid sizes of kernels that deliberately occupy
    // only part of the GPU); empty when every kernel spans the machine
    virtual std::string info() const { return std::string(); }
};

class Model {
public:
    virtual ~Model() = default;
    virtual size_t workspace_bytes(int N, int T_in) const = 0;
    // CudaCaller::variable_chunk_sizes (api/runner_creation.cpp:24-42): chunks of different lengths in one batch
    virtual bool variable_chunk_sizes() const { return false; }
    // How many runners (batches in flight) the engine expects to serve concurrently (Engine::set_num_runners).  Plans of
    // latency-bound kernels use it to size their grids: with R batches in flight a recurrence is better run on ~1/R of the
    // SMs with more chunks per CTA, side by side with the other batches' kernels, than spread thin over the whole GPU.
    int num_runners_hint = 2;
    virtual std::unique_ptr<ForwardPlan> make_plan(int N, int T_in, const __half* signal, __half* scores,
                                                   void* workspace, size_t workspace_bytes) = 0;
};

std::unique_ptr<Model> make_lstm_model(const b200_model_desc& desc, const b200_tensor* tensors, int n);
std::unique_ptr<Model> make_tx_model(const b200_model_desc& desc, const b200_tensor* tensors, int n);

// weight lookup helpers shared by the model builders
const b200_tensor& find_tensor(const b200_tensor* tensors, int n, const std::string& name);
// upload fp32 host data as fp16 / fp32 device arrays (freed with cudaFree by the owner)
__half* upload_f16(const std::vector<float>& v);
float* upload_f32(const std::vector<float>& v);

class Engine {
public:
    Engine(const b200_model_desc& desc, const b200_tensor* tensors, int num_tensors, int device);
    ~Engine();
    const b200_model_desc& desc() const { return m_desc; }
    int device() const { return m_device; }
    cudaStream_t stream() const { return m_stream; }
    Model& model() { return *m_model; }
    std::mutex& stats_mutex() { return m_stats_mutex; }  // guards the timing totals below
    b200_stats stats() const;

    // Lifecycle of CudaCaller (CudaCaller.cpp:126-138, 216-222, 273-287).  The reference parks a GPU worker thread per
    // caller; here calls run on the callers' own threads, so terminate() refuses new batches and waits for the ones in
    // flight, restart() (idempotent, callable once per runner sharing the engine) admits batches again.
    void terminate();
    void restart();
    bool terminated() const { return m_terminated.load(); }
    // Low-latency callers (adaptive sampling): 350 ms batch timeouts instead of 5 min / 30 s, and -- where the reference
    // gives them a task queue of their own (CudaCaller.cpp:204-214) -- their runners get CUDA streams of the highest
    // priority, so their kernels are scheduled ahead of the throughput runners sharing the GPU.  Set before creating runners.
    void set_low_latency(bool on) { m_low_latency.store(on); }
    // num_runners of api::create_basecall_runners (api/runner_creation.cpp:46-130; dorado's default is 2 per device): the
    // number of runners this engine is going to serve.  Set before creating runners; it only shapes launch plans.
    void set_num_runners(int n) { m_model->num_runners_hint = n < 1 ? 1 : (n > 16 ? 16 : n); }
    int num_runners() const { return m_model->num_runners_hint; }
    bool low_latency() const { return m_low_latency.load(); }
    void batch_timeouts_ms(int* first_chunk_ms, int* last_chunk_ms) const;
    struct CallGuard {  // brackets one call_chunks
        explicit CallGuard(Engine& e);
        ~CallGuard();
        Engine& eng;
    };

    std::atomic<int64_t> batches_called{0};
    std::atomic<int64_t> gpu_launches{0};
    std::atomic<int64_t> arena_bytes{0};
    double model_decode_ms = 0, h2d_ms = 0, d2h_ms = 0;  // guarded by stats_mutex

private:
    b200_model_desc m_desc;
    int m_device;
    cudaStream_t m_stream = nullptr;
    std::unique_ptr<Model> m_model;
    mutable std::mutex m_stats_mutex;
    std::atomic<bool> m_terminated{false};
    std::atomic<bool> m_low_latency{false};
    std::mutex m_life_mutex;
    std::condition_variable m_life_cv;
    int m_in_flight = 0;  // guarded by m_life_mutex
};

class Runner;
void pipelined_steps(Runner** runners, int n_runners, int num_chunks, int iters, float* total_ms);

// One runner = one batch in flight: its own stream, pinned host buffers, arena and launch plan (the reference's
// CudaModelRunner owns a stream too, CudaModelRunner.cpp:13-19).  Runners of one engine run concurrently.
class Runner {
public:
    friend void pipelined_steps(Runner** runners, int n_runners, int num_chunks, int iters, float* total_ms);
    Runner(Engine& engine, int batch_size, int chunk_size);
    ~Runner();
    int batch_size() const { return m_N; }
    int chunk_size() const { return m_T_in; }
    int out_len() const { return m_T_out; }
    // Direct access to the pinned fp16 batch.  Slots keep what they were given until they are given something else (as the
    // reference's input tensor does), so asking for the buffer turns every raw slot back into an fp16 slot: rows written
    // through the pointer are what the next call_chunks uploads.  Ask again after accept_raw_chunk before writing rows.
    uint16_t* input();
    void set_decoder_options(const b200_decoder_options& o);
    void accept_chunk_f16(int idx, const uint16_t* samples, int64_t len);
    void accept_chunk_f32(int idx, const float* samples, int64_t len);
    // variable chunk sizes (CudaModelRunner::accept_chunk, CudaModelRunner.cpp:21-31): len <= chunk_size, multiple of stride
    bool variable_chunk_sizes() const;
    void accept_chunk_var_f16(int idx, const uint16_t* samples, int64_t len);
    // raw int16 chunk: slice + scale + repeat-pad happen on the device (frontend.cu)
    void accept_raw_chunk(int idx, const b200_raw_chunk& chunk);
    void debug_read_input(int num_chunks, uint16_t* input_out);
    b200_result call_chunks(int num_chunks);
    void upload();
    void fill_synthetic_input();
    void step_device(int num_chunks, int iters, float* total_ms, float* forward_ms, float* decode_ms);
    void forward_scores_to_host(int num_chunks, uint16_t* scores_out);
    void debug_read_workspace(uint64_t offset, uint64_t bytes, void* dst);
    // one forward+decode pass with an event after every launch; returns "name=ms;name=ms;..."
    std::string profile(int num_chunks);
    std::string plan_info() const { return m_plan ? m_plan->info() : std::string(); }

private:
    void init();     // everything the constructor allocates; may throw
    void release();  // idempotent teardown shared by the destructor and a failed constructor
    bool m_counted = false;
    void stage_input(int n);  // H2D of the first n slots (+ gather/scale kernel for raw slots), on m_stream
    void clear_raw_slot(int idx);
    void run_forward(int n);
    void run_decode(int n, ProfileSink* prof = nullptr);

    Engine& m_engine;
    cudaStream_t m_stream = nullptr;
    std::mutex m_mutex;  // a runner is driven by one thread at a time
    int m_N, m_T_in, m_T_out, m_C;
    b200_decoder_options m_opts;
    // pinned host (input and output are separate allocations; the reference aliases them)
    uint16_t* m_h_input = nullptr;
    unsigned char* m_h_out = nullptr;  // moves | sequence | qstring | n_bases
    // raw-chunk staging (allocated on the first accept_raw_chunk): pinned int16 [N][T_in] + per-slot descriptors
    int16_t* m_h_raw = nullptr;
    RawSlot* m_h_slots = nullptr;
    int16_t* m_d_raw = nullptr;
    RawSlot* m_d_slots = nullptr;
    int m_num_raw = 0;  // slots currently holding a raw chunk
    // device
    Arena m_arena;
    __half* m_d_input = nullptr;
    __half* m_d_scores = nullptr;
    void* m_d_ws = nullptr;
    size_t m_ws_bytes = 0;
    std::unique_ptr<ForwardPlan> m_plan;
    float* m_d_bwd = nullptr;
    uint2* m_d_beam = nullptr;
    b200_qtable* m_d_qtable = nullptr;  // quality-character quantiser for (q_scale, q_shift), include/b200_crf_math.h
    void upload_qtable();
    unsigned char* m_d_out = nullptr;
    size_t m_out_bytes = 0;
    // variable chunk sizes: per-slot length in samples (pinned host + device) and the blocks each result row holds
    int32_t* m_h_lens = nullptr;
    int32_t* m_d_lens = nullptr;
    int32_t* m_h_nmoves = nullptr;
    cudaEvent_t m_ev[4] = {nullptr, nullptr, nullptr, nullptr};
};

// One process, several devices: see pool.cu.
class Pool {
public:
    Pool(const b200_model_desc& desc, const b200_tensor* tensors, int num_tensors, const int* devices, int num_devices,
         int runners_per_device, int batch_size, int chunk_size);
    ~Pool();
    int num_runners() const;
    Runner* runner(int i);
    int runner_numa_node(int i) const;
    int64_t runner_batches(int i) const;
    int out_len() const { return m_t_out; }
    // Feeds `num_chunks` host chunks (fp16 [num_chunks][chunk_size]) through all runners from a shared cursor; blocking.
    // Output rows have pitch out_len(); any output pointer may be null.  Returns wall seconds.
    double call_chunks(const uint16_t* chunks, int64_t num_chunks, uint8_t* moves, char* sequence, char* qstring,
                       int32_t* n_bases);

private:
    struct Worker;
    struct Job {
        const uint16_t* chunks = nullptr;
        int64_t num_chunks = 0;
        uint8_t* moves = nullptr;
        char* sequence = nullptr;
        char* qstring = nullptr;
        int32_t* n_bases = nullptr;
    };
    void worker_main(Worker& w);
    void shutdown();
    int m_batch, m_chunk, m_t_out = 0;
    std::vector<std::unique_ptr<Engine>> m_engines;
    std::vector<std::unique_ptr<Worker>> m_workers;
    std::mutex m_mutex, m_job_mutex;
    std::condition_variable m_cv_job, m_cv_done;
    long long m_job_id = 0;
    int m_ready = 0, m_done = 0;
    bool m_stop = false;
    Job m_job;
    std::atomic<int64_t> m_cursor{0};
};

void decode_host_scores(int device, const uint16_t* scores, int N, int T, int C, float clamp_val,
                        const b200_decoder_options& opts, uint8_t* moves, char* sequence, char* qstring,
                        int32_t* n_bases);
void test_gemm_host(int device, const uint16_t* a, const uint16_t* b, const float* bias, int M, int N, int K,
                    int activation, uint16_t* c);

// batch-size selection (CudaCaller::determine_batch_dims)
size_t runner_device_bytes(Engine& engine, int batch_size, int chunk_size);
int benchmark_batch_sizes(Engine& engine, int chunk_size, int granularity, int max_batch_size, int32_t* batch_sizes,
                          float* ms_per_chunk, int capacity);
int select_batch_size(const int32_t* batch_sizes, const float* ms_per_chunk, int count, int max_batch_size, int granularity,
                      float time_penalty);

// pre-computed batch-size timings (CudaChunkBenchmarks): rows found for (gpu, model), 0 if there is no table
int lookup_chunk_benchmarks(const char* gpu_name, const char* model_name, int32_t* batch_sizes, float* ms_per_chunk, int capacity);
std::string device_name(int device);

// cudaFuncAttributeMaxDynamicSharedMemorySize is per device and per function: set it once for each (device, kernel)
// pair, from whichever thread gets there first (several runners, and in dorado several devices, share one process).
void ensure_dynamic_smem(const void* kernel, int bytes);
template <typename K>
inline void ensure_dynamic_smem(K* kernel, int bytes) {
    ensure_dynamic_smem(reinterpret_cast<const void*>(kernel), bytes);
}

float log_beam_cut_of(float beam_cut);
void require_sm90(int device);

}  // namespace b200
