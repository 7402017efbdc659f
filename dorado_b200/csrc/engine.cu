// Engine / Runner: see engine.h.  Mirrors the control flow of the reference's CudaCaller::call_chunks
// (dorado/basecall/CudaCaller.cpp:224-271): H2D copy, forward, decode part 1 on the GPU, D2H of the
// 3 x N x T byte result -- here without libtorch, Koi or a separate GPU worker thread.  Every runner has its own stream,
// so the runners of a device overlap (one batch's decode under the next batch's network) instead of queueing behind
// the reference's per-device task queue (CudaCaller.cpp:204-214).
#include "engine.h"

#include "b200_crf_math.h"
#include "decode.h"
#include "nvtx.h"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <cstring>
#include <limits>
#include <set>
#include <utility>
#include <vector>

namespace b200 {

Arena::~Arena() {
    if (m_base) cudaFree(m_base);
}

void Arena::reserve(size_t bytes) {
    if (m_base) throw std::logic_error("Arena::reserve called twice");
    B200_CUDA(cudaMalloc(&m_base, bytes));
    m_cap = bytes;
    m_off = 0;
}

void* Arena::take(size_t bytes) {
    const size_t aligned = (bytes + 255) & ~size_t(255);
    if (m_off + aligned > m_cap) throw std::logic_error("Arena overflow");
    void* p = m_base + m_off;
    m_off += aligned;
    return p;
}

void ensure_dynamic_smem(const void* kernel, int bytes) {
    static std::mutex mu;
    static std::set<std::pair<int, const void*>> done;
    int dev = 0;
    B200_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lock(mu);
    if (done.count({dev, kernel})) return;
    B200_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    done.insert({dev, kernel});
}

// byte offset of the int32 n_bases array behind the three [N][T] byte planes
static size_t nb_offset(int N, int T) { return ((size_t)3 * N * T + 15) & ~size_t(15); }

const b200_tensor& find_tensor(const b200_tensor* tensors, int n, const std::string& name) {
    for (int i = 0; i < n; ++i) {
        if (tensors[i].name && name == tensors[i].name) return tensors[i];
    }
    throw std::invalid_argument("missing weight tensor '" + name + "'");
}

__half* upload_f16(const std::vector<float>& v) {
    std::vector<__half> h(v.size());
    for (size_t i = 0; i < v.size(); ++i) h[i] = __float2half_rn(v[i]);
    __half* d = nullptr;
    B200_CUDA(cudaMalloc(&d, h.size() * sizeof(__half) + 16));
    B200_CUDA(cudaMemcpy(d, h.data(), h.size() * sizeof(__half), cudaMemcpyHostToDevice));
    return d;
}

float* upload_f32(const std::vector<float>& v) {
    float* d = nullptr;
    B200_CUDA(cudaMalloc(&d, v.size() * sizeof(float) + 16));
    B200_CUDA(cudaMemcpy(d, v.data(), v.size() * sizeof(float), cudaMemcpyHostToDevice));
    return d;
}

float log_beam_cut_of(float beam_cut) {
    // beam_search.cpp:147-148
    return beam_cut > 0.0f ? logf(beam_cut) : std::numeric_limits<float>::max();
}

void require_sm90(int device) {
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) {
        cudaGetLastError();
        throw CudaError("b200call: no CUDA device visible; this library has no CPU fallback");
    }
    if (device < 0 || device >= count) throw std::invalid_argument("b200call: bad device index");
    cudaDeviceProp prop{};
    B200_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {
        throw CudaError(std::string("b200call: device '") + prop.name + "' is sm_" + std::to_string(prop.major) +
                        std::to_string(prop.minor) + "; this build contains sm_90a code only");
    }
    B200_CUDA(cudaSetDevice(device));
}

Engine::Engine(const b200_model_desc& desc, const b200_tensor* tensors, int num_tensors, int device)
        : m_desc(desc), m_device(device) {
    if (desc.state_len < 3 || desc.state_len > 5) throw std::invalid_argument("state_len must be 3..5");
    if (desc.outsize != (1 << (2 * (desc.state_len + 1)))) throw std::invalid_argument("outsize != 4^(state_len+1)");
    if (desc.num_convs < 1 || desc.num_convs > 8) throw std::invalid_argument("num_convs must be in [1, 8]");
    if (desc.stride < 1) throw std::invalid_argument("stride must be positive");
    require_sm90(device);
    B200_CUDA(cudaStreamCreateWithFlags(&m_stream, cudaStreamNonBlocking));
    if (desc.model_type == B200_MODEL_LSTM) {
        m_model = make_lstm_model(desc, tensors, num_tensors);
    } else if (desc.model_type == B200_MODEL_TX) {
        m_model = make_tx_model(desc, tensors, num_tensors);
    } else {
        throw std::invalid_argument("unknown model_type");
    }
}

Engine::~Engine() {
    cudaSetDevice(m_device);
    m_model.reset();
    if (m_stream) cudaStreamDestroy(m_stream);
}

void Engine::terminate() {
    m_terminated.store(true);
    std::unique_lock<std::mutex> lock(m_life_mutex);
    m_life_cv.wait(lock, [&] { return m_in_flight == 0; });
}

void Engine::restart() { m_terminated.store(false); }

void Engine::batch_timeouts_ms(int* first_chunk_ms, int* last_chunk_ms) const {
    // CudaCaller.cpp:121-138, 216-222
    const bool ll = m_low_latency.load();
    if (first_chunk_ms) *first_chunk_ms = ll ? 350 : 300000;
    if (last_chunk_ms) *last_chunk_ms = ll ? 350 : 30000;
}

Engine::CallGuard::CallGuard(Engine& e) : eng(e) {
    std::lock_guard<std::mutex> lock(e.m_life_mutex);
    if (e.m_terminated.load()) throw std::logic_error("call_chunks on a terminated caller (restart() it first)");
    ++e.m_in_flight;
}

Engine::CallGuard::~CallGuard() {
    {
        std::lock_guard<std::mutex> lock(eng.m_life_mutex);
        --eng.m_in_flight;
    }
    eng.m_life_cv.notify_all();
}

b200_stats Engine::stats() const {
    b200_stats s{};
    std::lock_guard<std::mutex> lock(m_stats_mutex);
    s.batches_called = batches_called.load();
    s.model_decode_ms = model_decode_ms;
    s.h2d_ms = h2d_ms;
    s.d2h_ms = d2h_ms;
    s.gpu_launches = gpu_launches.load();
    s.arena_bytes = arena_bytes.load();
    return s;
}

Runner::Runner(Engine& engine, int batch_size, int chunk_size) : m_engine(engine), m_N(batch_size), m_T_in(chunk_size) {
    try {
        init();
    } catch (...) {
        release();  // the destructor does not run for a half-built object: hand back pinned memory, stream, events
        throw;
    }
    // only a fully built runner is charged to the engine's statistics
    engine.arena_bytes += (int64_t)m_arena.capacity();
    m_counted = true;
}

void Runner::init() {
    Engine& engine = m_engine;
    const int batch_size = m_N, chunk_size = m_T_in;
    const auto& d = engine.desc();
    if (batch_size < 1) throw std::invalid_argument("batch_size must be >= 1");
    const int stride_inner = d.model_type == B200_MODEL_TX ? d.stride * d.upsample_scale : d.stride;
    const int gran = d.model_type == B200_MODEL_TX ? stride_inner * 16 : d.stride;
    if (chunk_size < gran || chunk_size % gran != 0) {
        // BatchParams::normalise (dorado/config/BatchParams.cpp:89-105) is the caller's job
        throw std::invalid_argument("chunk_size must be a positive multiple of " + std::to_string(gran));
    }
    m_T_out = chunk_size / d.stride;
    if ((size_t)m_T_out > decode_max_blocks()) {
        throw std::invalid_argument("chunk_size / stride = " + std::to_string(m_T_out) + " blocks exceed the decoder's limit of " +
                                    std::to_string(decode_max_blocks()));
    }
    m_C = d.outsize;
    b200_default_decoder_options(&m_opts);
    m_opts.q_scale = d.qscale;
    m_opts.q_shift = d.qbias;

    B200_CUDA(cudaSetDevice(engine.device()));
    {
        int least = 0, greatest = 0;  // numerically lowest value = highest priority
        B200_CUDA(cudaDeviceGetStreamPriorityRange(&least, &greatest));
        B200_CUDA(cudaStreamCreateWithPriority(&m_stream, cudaStreamNonBlocking, engine.low_latency() ? greatest : least));
    }
    const size_t in_bytes = (size_t)m_N * m_T_in * sizeof(uint16_t);
    m_out_bytes = nb_offset(m_N, m_T_out) + (size_t)m_N * sizeof(int32_t);
    B200_CUDA(cudaHostAlloc(&m_h_input, in_bytes, cudaHostAllocDefault));
    std::memset(m_h_input, 0, in_bytes);
    B200_CUDA(cudaHostAlloc(&m_h_out, m_out_bytes, cudaHostAllocDefault));
    B200_CUDA(cudaHostAlloc(&m_h_lens, (size_t)2 * m_N * sizeof(int32_t), cudaHostAllocDefault));
    m_h_nmoves = m_h_lens + m_N;
    for (int i = 0; i < m_N; ++i) {
        m_h_lens[i] = m_T_in;
        m_h_nmoves[i] = m_T_out;
    }

    size_t bwd_b = 0, beam_b = 0;
    decode_scratch_bytes(m_N, m_T_out, d.state_len, &bwd_b, &beam_b);
    const size_t scores_b = (size_t)m_N * m_T_out * m_C * sizeof(__half);
    const size_t ws_b = engine.model().workspace_bytes(m_N, m_T_in);
    auto al = [](size_t b) { return (b + 255) & ~size_t(255); };
    const size_t lens_b = engine.model().variable_chunk_sizes() ? (size_t)m_N * sizeof(int32_t) : 0;
    m_arena.reserve(al(in_bytes) + al(scores_b) + al(ws_b) + al(bwd_b) + al(beam_b) + al(m_out_bytes) + al(lens_b) + 4096);
    m_d_qtable = static_cast<b200_qtable*>(m_arena.take(sizeof(b200_qtable)));  // inside the 4096 bytes of slack
    if (lens_b) m_d_lens = static_cast<int32_t*>(m_arena.take(lens_b));
    m_d_input = static_cast<__half*>(m_arena.take(in_bytes));
    m_d_scores = static_cast<__half*>(m_arena.take(scores_b));
    m_d_ws = m_arena.take(ws_b);
    m_ws_bytes = ws_b;
    m_d_bwd = static_cast<float*>(m_arena.take(bwd_b));
    m_d_beam = static_cast<uint2*>(m_arena.take(beam_b));
    m_d_out = static_cast<unsigned char*>(m_arena.take(m_out_bytes));
    // zero padding rows / unused slots once, on the engine's own (non-blocking) stream so it is ordered
    // before the first forward
    B200_CUDA(cudaMemsetAsync(m_d_input, 0, in_bytes, m_stream));
    B200_CUDA(cudaMemsetAsync(m_d_ws, 0, ws_b, m_stream));
    B200_CUDA(cudaStreamSynchronize(m_stream));
    m_plan = engine.model().make_plan(m_N, m_T_in, m_d_input, m_d_scores, m_d_ws, ws_b);
    if (m_d_lens) {
        B200_CUDA(cudaMemcpyAsync(m_d_lens, m_h_lens, (size_t)m_N * sizeof(int32_t), cudaMemcpyHostToDevice, m_stream));
        B200_CUDA(cudaStreamSynchronize(m_stream));
        m_plan->set_chunk_lengths(m_d_lens);
    }
    for (auto& e : m_ev) B200_CUDA(cudaEventCreate(&e));
    upload_qtable();
}

// The per-base quality character is a quantiser of err = 1 - p_called / p_total (beam_search.cpp:94-98); its bin edges
// are placed on the host with the host's own log10f, so the device reproduces the reference's characters exactly.
void Runner::upload_qtable() {
    b200_qtable tb;
    if (b200_qtable_build(m_opts.q_scale, m_opts.q_shift, &tb) != 0) {
        throw std::invalid_argument("decoder options: q_scale and q_shift must be finite");
    }
    B200_CUDA(cudaSetDevice(m_engine.device()));
    B200_CUDA(cudaMemcpyAsync(m_d_qtable, &tb, sizeof(tb), cudaMemcpyHostToDevice, m_stream));
    B200_CUDA(cudaStreamSynchronize(m_stream));
}

Runner::~Runner() { release(); }

void Runner::release() {
    cudaSetDevice(m_engine.device());
    if (m_stream) cudaStreamSynchronize(m_stream);
    if (m_counted) m_engine.arena_bytes -= (int64_t)m_arena.capacity();
    if (m_h_raw) m_engine.arena_bytes -= (int64_t)((size_t)m_N * m_T_in * sizeof(int16_t) + (size_t)m_N * sizeof(RawSlot));
    m_counted = false;
    for (auto& e : m_ev) {
        if (e) cudaEventDestroy(e);
        e = nullptr;
    }
    m_plan.reset();
    if (m_h_input) cudaFreeHost(m_h_input);
    if (m_h_out) cudaFreeHost(m_h_out);
    if (m_h_lens) cudaFreeHost(m_h_lens);
    m_h_lens = nullptr;
    m_h_nmoves = nullptr;
    if (m_h_raw) cudaFreeHost(m_h_raw);
    if (m_h_slots) cudaFreeHost(m_h_slots);
    if (m_d_raw) cudaFree(m_d_raw);
    if (m_d_slots) cudaFree(m_d_slots);
    m_h_input = nullptr;
    m_h_out = nullptr;
    m_h_raw = nullptr;
    m_h_slots = nullptr;
    m_d_raw = nullptr;
    m_d_slots = nullptr;
    if (m_stream) cudaStreamDestroy(m_stream);
    m_stream = nullptr;
}

void Runner::set_decoder_options(const b200_decoder_options& o) {
    if (o.beam_width < 1 || o.beam_width > 32) throw std::invalid_argument("beam_width must be in [1, 32]");
    if (o.move_pad != 0) throw Unsupported("move_pad: only the closed Koi kernel defines it; the reference never sets it");
    if (o.temperature != 1.0f) throw Unsupported("temperature != 1: no decoder of the reference reads this option");
    std::lock_guard<std::mutex> lock(m_mutex);
    m_opts = o;
    upload_qtable();
}

void Runner::accept_chunk_f16(int idx, const uint16_t* samples, int64_t len) {
    if (idx < 0 || idx >= m_N) throw std::invalid_argument("accept_chunk: chunk_idx out of range");
    if (len != m_T_in) throw std::invalid_argument("accept_chunk: chunk length != chunk_size");
    std::lock_guard<std::mutex> lock(m_mutex);
    clear_raw_slot(idx);
    std::memcpy(m_h_input + (size_t)idx * m_T_in, samples, (size_t)len * sizeof(uint16_t));
    m_h_lens[idx] = m_T_in;
    m_h_nmoves[idx] = m_T_out;
}

bool Runner::variable_chunk_sizes() const { return m_d_lens != nullptr; }

void Runner::accept_chunk_var_f16(int idx, const uint16_t* samples, int64_t len) {
    if (idx < 0 || idx >= m_N) throw std::invalid_argument("accept_chunk: chunk_idx out of range");
    if (!m_d_lens) throw Unsupported("this model has no variable-chunk-size mode (b200_runner_variable_chunk_sizes() == 0)");
    const int stride = m_engine.desc().stride;
    if (len < stride || len > m_T_in || len % stride != 0) {
        throw std::invalid_argument("accept_chunk: a variable chunk must be a positive multiple of the stride, <= chunk_size");
    }
    std::lock_guard<std::mutex> lock(m_mutex);
    clear_raw_slot(idx);
    std::memcpy(m_h_input + (size_t)idx * m_T_in, samples, (size_t)len * sizeof(uint16_t));
    m_h_lens[idx] = (int32_t)len;
    m_h_nmoves[idx] = (int32_t)(len / stride);
}

void Runner::accept_chunk_f32(int idx, const float* samples, int64_t len) {
    if (idx < 0 || idx >= m_N) throw std::invalid_argument("accept_chunk: chunk_idx out of range");
    if (len != m_T_in) throw std::invalid_argument("accept_chunk: chunk length != chunk_size");
    std::lock_guard<std::mutex> lock(m_mutex);
    clear_raw_slot(idx);
    __half* dst = reinterpret_cast<__half*>(m_h_input + (size_t)idx * m_T_in);
    for (int64_t i = 0; i < len; ++i) dst[i] = __float2half_rn(samples[i]);
    m_h_lens[idx] = m_T_in;
    m_h_nmoves[idx] = m_T_out;
}

uint16_t* Runner::input() {
    std::lock_guard<std::mutex> lock(m_mutex);
    if (m_num_raw > 0) {
        for (int i = 0; i < m_N; ++i) m_h_slots[i].slice_len = 0;
        m_num_raw = 0;
    }
    return m_h_input;
}

void Runner::clear_raw_slot(int idx) {
    if (m_h_slots && m_h_slots[idx].slice_len > 0) {
        m_h_slots[idx].slice_len = 0;
        --m_num_raw;
    }
}

// BasecallerNode's input slice (BasecallerNode.cpp:395-400): raw[offset : offset + chunk_size], clamped at the read
// end.  Only the slice is staged; scaling and repeat-padding happen on the device (frontend.cu).
void Runner::accept_raw_chunk(int idx, const b200_raw_chunk& c) {
    if (idx < 0 || idx >= m_N) throw std::invalid_argument("accept_raw_chunk: chunk_idx out of range");
    if (!c.raw || c.num_samples == 0) throw std::invalid_argument("accept_raw_chunk: empty read");
    if (c.input_offset >= c.num_samples) throw std::invalid_argument("accept_raw_chunk: input_offset beyond the read");
    if (!(c.scale != 0.0f) || c.scale != c.scale || c.shift != c.shift) {
        throw std::invalid_argument("accept_raw_chunk: scale must be non-zero and finite");
    }
    std::lock_guard<std::mutex> lock(m_mutex);
    if (!m_h_raw) {
        B200_CUDA(cudaSetDevice(m_engine.device()));
        const size_t raw_b = (size_t)m_N * m_T_in * sizeof(int16_t);
        B200_CUDA(cudaHostAlloc(&m_h_raw, raw_b, cudaHostAllocDefault));
        B200_CUDA(cudaHostAlloc(&m_h_slots, (size_t)m_N * sizeof(RawSlot), cudaHostAllocDefault));
        std::memset(m_h_raw, 0, raw_b);
        std::memset(m_h_slots, 0, (size_t)m_N * sizeof(RawSlot));
        B200_CUDA(cudaMalloc(&m_d_raw, raw_b));
        B200_CUDA(cudaMalloc(&m_d_slots, (size_t)m_N * sizeof(RawSlot)));
        m_engine.arena_bytes += (int64_t)(raw_b + (size_t)m_N * sizeof(RawSlot));
    }
    const uint64_t avail = c.num_samples - c.input_offset;
    const int slice = (int)std::min<uint64_t>(avail, (uint64_t)m_T_in);
    std::memcpy(m_h_raw + (size_t)idx * m_T_in, c.raw + c.input_offset, (size_t)slice * sizeof(int16_t));
    if (m_h_slots[idx].slice_len == 0) ++m_num_raw;
    m_h_slots[idx].slice_len = slice;
    m_h_slots[idx].shift = c.shift;
    m_h_slots[idx].scale = c.scale;
    m_h_lens[idx] = m_T_in;
    m_h_nmoves[idx] = m_T_out;
}

// Input stage of a batch: fp16 rows by plain H2D; raw rows as staged int16 + descriptors, then one gather/scale
// kernel writes their fp16 rows (it skips fp16 slots, so both kinds can share a batch).
void Runner::stage_input(int n) {
    if (m_d_lens) {
        B200_CUDA(cudaMemcpyAsync(m_d_lens, m_h_lens, (size_t)m_N * sizeof(int32_t), cudaMemcpyHostToDevice, m_stream));
    }
    int raw_in_n = 0;
    if (m_num_raw > 0) {
        for (int i = 0; i < n; ++i) raw_in_n += m_h_slots[i].slice_len > 0;
    }
    if (raw_in_n < n) {
        B200_CUDA(cudaMemcpyAsync(m_d_input, m_h_input, (size_t)n * m_T_in * sizeof(uint16_t), cudaMemcpyHostToDevice,
                                  m_stream));
    }
    if (raw_in_n > 0) {
        B200_CUDA(cudaMemcpyAsync(m_d_raw, m_h_raw, (size_t)n * m_T_in * sizeof(int16_t), cudaMemcpyHostToDevice, m_stream));
        B200_CUDA(cudaMemcpyAsync(m_d_slots, m_h_slots, (size_t)n * sizeof(RawSlot), cudaMemcpyHostToDevice, m_stream));
        launch_raw_chunk_gather(m_d_raw, m_d_slots, m_d_input, n, m_T_in, m_stream);
        ++m_engine.gpu_launches;
    }
}

void Runner::debug_read_input(int num_chunks, uint16_t* input_out) {
    if (num_chunks < 1 || num_chunks > m_N || !input_out) throw std::invalid_argument("debug_read_input: bad arguments");
    std::lock_guard<std::mutex> lock(m_mutex);
    B200_CUDA(cudaSetDevice(m_engine.device()));
    stage_input(num_chunks);
    B200_CUDA(cudaMemcpyAsync(input_out, m_d_input, (size_t)num_chunks * m_T_in * sizeof(uint16_t), cudaMemcpyDeviceToHost,
                              m_stream));
    B200_CUDA(cudaStreamSynchronize(m_stream));
}

void Runner::run_forward(int n) {
    (void)n;  // the whole batch is computed; only the first n chunks are decoded and returned
    NvtxRange range("nn_forward");
    m_plan->run(m_stream);
    m_engine.gpu_launches += m_plan->launches();
}

void Runner::run_decode(int n, ProfileSink* prof) {
    NvtxRange range("gpu_decode");
    const auto& d = m_engine.desc();
    DecodeArgs a{};
    a.scores = m_d_scores;
    a.N = n;
    a.T = m_T_out;
    a.state_len = d.state_len;
    a.clamp_val = d.clamp ? 5.0f : 0.0f;  // decode/Decoder.cpp:19
    a.beam_width = m_opts.beam_width;
    a.log_beam_cut = log_beam_cut_of(m_opts.beam_cut);
    a.blank = m_opts.blank_score;
    a.q_shift = m_opts.q_shift;
    a.q_scale = m_opts.q_scale;
    a.qtable = m_d_qtable;
    a.lens = m_d_lens;
    a.stride = d.stride;
    a.bwd = m_d_bwd;
    a.beam = m_d_beam;
    // output rows are packed for the n chunks actually called
    a.moves = m_d_out;
    a.sequence = reinterpret_cast<char*>(m_d_out + (size_t)m_N * m_T_out);
    a.qstring = reinterpret_cast<char*>(m_d_out + (size_t)2 * m_N * m_T_out);
    a.n_bases = reinterpret_cast<int32_t*>(m_d_out + nb_offset(m_N, m_T_out));
    decode_scores(a, m_stream, prof);
    m_engine.gpu_launches += 3;
}

// Deterministic pseudo-random fp16 signal in [-2, 2) for the batch-size benchmark (an LCG: no <random> state to share).
void Runner::fill_synthetic_input() {
    std::lock_guard<std::mutex> lock(m_mutex);
    uint32_t x = 0x2545f491u;
    __half* dst = reinterpret_cast<__half*>(m_h_input);
    for (size_t i = 0; i < (size_t)m_N * m_T_in; ++i) {
        x = x * 1664525u + 1013904223u;
        dst[i] = __float2half_rn((float)(int32_t)(x >> 8 & 0xffff) * (4.0f / 65536.0f) - 2.0f);
    }
    B200_CUDA(cudaSetDevice(m_engine.device()));
    stage_input(m_N);
    B200_CUDA(cudaStreamSynchronize(m_stream));
}

void Runner::upload() {
    std::lock_guard<std::mutex> lock(m_mutex);
    B200_CUDA(cudaSetDevice(m_engine.device()));
    stage_input(m_N);
    B200_CUDA(cudaStreamSynchronize(m_stream));
}

b200_result Runner::call_chunks(int num_chunks) {
    if (num_chunks < 1 || num_chunks > m_N) throw std::invalid_argument("call_chunks: num_chunks out of range");
    NvtxRange range("call_chunks");  // CudaCaller::call_chunks, NVTX3_FUNC_RANGE (CudaCaller.cpp:228)
    Engine::CallGuard in_flight(m_engine);
    std::lock_guard<std::mutex> lock(m_mutex);
    B200_CUDA(cudaSetDevice(m_engine.device()));
    cudaStream_t s = m_stream;
    B200_CUDA(cudaEventRecord(m_ev[0], s));
    stage_input(num_chunks);
    B200_CUDA(cudaEventRecord(m_ev[1], s));
    run_forward(num_chunks);
    run_decode(num_chunks);
    B200_CUDA(cudaEventRecord(m_ev[2], s));
    B200_CUDA(cudaMemcpyAsync(m_h_out, m_d_out, m_out_bytes, cudaMemcpyDeviceToHost, s));
    B200_CUDA(cudaEventRecord(m_ev[3], s));
    B200_CUDA(cudaStreamSynchronize(s));
    float h2d = 0, md = 0, d2h = 0;
    B200_CUDA(cudaEventElapsedTime(&h2d, m_ev[0], m_ev[1]));
    B200_CUDA(cudaEventElapsedTime(&md, m_ev[1], m_ev[2]));
    B200_CUDA(cudaEventElapsedTime(&d2h, m_ev[2], m_ev[3]));
    {
        std::lock_guard<std::mutex> sl(m_engine.stats_mutex());
        m_engine.h2d_ms += h2d;
        m_engine.model_decode_ms += md;
        m_engine.d2h_ms += d2h;
    }
    ++m_engine.batches_called;
    b200_result r{};
    r.moves = m_h_out;
    r.sequence = reinterpret_cast<const char*>(m_h_out + (size_t)m_N * m_T_out);
    r.qstring = reinterpret_cast<const char*>(m_h_out + (size_t)2 * m_N * m_T_out);
    r.n_bases = reinterpret_cast<const int32_t*>(m_h_out + nb_offset(m_N, m_T_out));
    r.t_out = m_T_out;
    r.num_chunks = num_chunks;
    r.n_moves = m_h_nmoves;
    return r;
}

void Runner::step_device(int num_chunks, int iters, float* total_ms, float* forward_ms, float* decode_ms) {
    if (num_chunks < 1 || num_chunks > m_N || iters < 1) throw std::invalid_argument("step_device: bad arguments");
    std::lock_guard<std::mutex> lock(m_mutex);
    B200_CUDA(cudaSetDevice(m_engine.device()));
    cudaStream_t s = m_stream;
    float fwd = 0, dec = 0;
    for (int i = 0; i < iters; ++i) {
        B200_CUDA(cudaEventRecord(m_ev[0], s));
        run_forward(num_chunks);
        B200_CUDA(cudaEventRecord(m_ev[1], s));
        run_decode(num_chunks);
        B200_CUDA(cudaEventRecord(m_ev[2], s));
        B200_CUDA(cudaStreamSynchronize(s));
        float ms = 0;
        B200_CUDA(cudaEventElapsedTime(&ms, m_ev[0], m_ev[1]));
        fwd += ms;
        B200_CUDA(cudaEventElapsedTime(&ms, m_ev[1], m_ev[2]));
        dec += ms;
    }
    *total_ms = fwd + dec;
    if (forward_ms) *forward_ms = fwd;
    if (decode_ms) *decode_ms = dec;
}

// Device-resident throughput with several runners in flight (the reference runs num_runners = 2 CudaModelRunners
// per device, api/runner_creation.cpp:91-123, so one runner's decode overlaps the next one's network).  Step i goes
// to runner i % R on that runner's own stream; the region is bracketed by events on runner 0's stream, which first
// releases and finally joins the other streams.
void pipelined_steps(Runner** rs, int R, int num_chunks, int iters, float* total_ms) {
    if (R < 1 || !rs || iters < 1) throw std::invalid_argument("pipelined_steps: bad arguments");
    for (int r = 0; r < R; ++r) {
        if (!rs[r]) throw std::invalid_argument("pipelined_steps: null runner");
        if (&rs[r]->m_engine != &rs[0]->m_engine) throw std::invalid_argument("pipelined_steps: runners of different engines");
        if (num_chunks < 1 || num_chunks > rs[r]->m_N) throw std::invalid_argument("pipelined_steps: num_chunks out of range");
        for (int q = 0; q < r; ++q) {
            if (rs[q] == rs[r]) throw std::invalid_argument("pipelined_steps: the same runner twice");
        }
    }
    std::vector<Runner*> order(rs, rs + R);
    std::sort(order.begin(), order.end());  // one global lock order, whatever order the callers list the runners in
    std::vector<std::unique_lock<std::mutex>> locks;
    for (Runner* r : order) locks.emplace_back(r->m_mutex);
    Runner& r0 = *rs[0];
    B200_CUDA(cudaSetDevice(r0.m_engine.device()));
    B200_CUDA(cudaEventRecord(r0.m_ev[0], r0.m_stream));
    for (int r = 1; r < R; ++r) B200_CUDA(cudaStreamWaitEvent(rs[r]->m_stream, r0.m_ev[0], 0));
    for (int i = 0; i < iters; ++i) {
        Runner& ru = *rs[i % R];
        ru.run_forward(num_chunks);
        ru.run_decode(num_chunks);
    }
    for (int r = 1; r < R; ++r) {
        B200_CUDA(cudaEventRecord(rs[r]->m_ev[2], rs[r]->m_stream));
        B200_CUDA(cudaStreamWaitEvent(r0.m_stream, rs[r]->m_ev[2], 0));
    }
    B200_CUDA(cudaEventRecord(r0.m_ev[1], r0.m_stream));
    B200_CUDA(cudaStreamSynchronize(r0.m_stream));
    B200_CUDA(cudaEventElapsedTime(total_ms, r0.m_ev[0], r0.m_ev[1]));
}

void Runner::forward_scores_to_host(int num_chunks, uint16_t* scores_out) {
    if (num_chunks < 1 || num_chunks > m_N) throw std::invalid_argument("forward_scores: num_chunks out of range");
    std::lock_guard<std::mutex> lock(m_mutex);
    B200_CUDA(cudaSetDevice(m_engine.device()));
    cudaStream_t s = m_stream;
    stage_input(num_chunks);
    run_forward(num_chunks);
    B200_CUDA(cudaMemcpyAsync(scores_out, m_d_scores, (size_t)num_chunks * m_T_out * m_C * sizeof(__half),
                              cudaMemcpyDeviceToHost, s));
    B200_CUDA(cudaStreamSynchronize(s));
}

void ProfileSink::begin(cudaStream_t s) { mark("begin", s); }

void ProfileSink::mark(const char* name, cudaStream_t s) {
    cudaEvent_t e;
    B200_CUDA(cudaEventCreate(&e));
    B200_CUDA(cudaEventRecord(e, s));
    events.push_back(e);
    names.emplace_back(name);
}

std::vector<std::pair<std::string, float>> ProfileSink::report() {
    std::vector<std::pair<std::string, float>> out;
    for (size_t i = 1; i < events.size(); ++i) {
        float ms = 0;
        B200_CUDA(cudaEventElapsedTime(&ms, events[i - 1], events[i]));
        out.emplace_back(names[i], ms);
    }
    return out;
}

ProfileSink::~ProfileSink() {
    for (auto e : events) cudaEventDestroy(e);
}

std::string Runner::profile(int num_chunks) {
    if (num_chunks < 1 || num_chunks > m_N) throw std::invalid_argument("profile: num_chunks out of range");
    std::lock_guard<std::mutex> lock(m_mutex);
    B200_CUDA(cudaSetDevice(m_engine.device()));
    cudaStream_t s = m_stream;
    ProfileSink sink;
    sink.begin(s);
    m_plan->run(s, &sink);
    m_engine.gpu_launches += m_plan->launches();
    run_decode(num_chunks, &sink);
    B200_CUDA(cudaStreamSynchronize(s));
    std::string out;
    for (auto& kv : sink.report()) out += kv.first + "=" + std::to_string(kv.second) + ";";
    return out;
}

void Runner::debug_read_workspace(uint64_t offset, uint64_t bytes, void* dst) {
    if (offset + bytes > m_ws_bytes) throw std::invalid_argument("debug_read_workspace: out of range");
    std::lock_guard<std::mutex> lock(m_mutex);
    B200_CUDA(cudaSetDevice(m_engine.device()));
    B200_CUDA(cudaStreamSynchronize(m_stream));
    B200_CUDA(cudaMemcpy(dst, static_cast<unsigned char*>(m_d_ws) + offset, bytes, cudaMemcpyDeviceToHost));
}

// ---- batch-size selection ------------------------------------------------------------------------------------------
// Same arithmetic as the Runner constructor's arena reservation (checked against b200_stats.arena_bytes on the GPU).
size_t runner_device_bytes(Engine& engine, int batch_size, int chunk_size) {
    const auto& d = engine.desc();
    if (batch_size < 1 || chunk_size < d.stride || chunk_size % d.stride != 0) {
        throw std::invalid_argument("runner_device_bytes: bad batch or chunk size");
    }
    const int T_out = chunk_size / d.stride;
    const size_t in_bytes = (size_t)batch_size * chunk_size * sizeof(uint16_t);
    const size_t out_bytes = nb_offset(batch_size, T_out) + (size_t)batch_size * sizeof(int32_t);
    size_t bwd_b = 0, beam_b = 0;
    decode_scratch_bytes(batch_size, T_out, d.state_len, &bwd_b, &beam_b);
    const size_t scores_b = (size_t)batch_size * T_out * d.outsize * sizeof(__half);
    const size_t ws_b = engine.model().workspace_bytes(batch_size, chunk_size);
    auto al = [](size_t b) { return (b + 255) & ~size_t(255); };
    const size_t lens_b = engine.model().variable_chunk_sizes() ? (size_t)batch_size * sizeof(int32_t) : 0;
    return al(in_bytes) + al(scores_b) + al(ws_b) + al(bwd_b) + al(beam_b) + al(out_bytes) + al(lens_b) + 4096;
}

int benchmark_batch_sizes(Engine& engine, int chunk_size, int granularity, int max_batch_size, int32_t* batch_sizes,
                          float* ms_per_chunk, int capacity) {
    if (granularity < 1 || max_batch_size < granularity) throw std::invalid_argument("benchmark_batch_sizes: bad range");
    int count = 0;
    for (int bs = granularity; bs <= max_batch_size; bs += granularity, ++count) {
        float best = std::numeric_limits<float>::max();
        {
            Runner scratch(engine, bs, chunk_size);
            scratch.fill_synthetic_input();  // beam-search time depends on the data: time a non-degenerate signal
            for (int i = 0; i < 2; ++i) {            // run twice to eliminate outliers (CudaCaller.cpp:536)
                float total = 0, fwd = 0, dec = 0;
                scratch.step_device(bs, 1, &total, &fwd, &dec);
                best = std::min(best, total / (float)bs);
            }
        }
        if (count < capacity) {
            if (batch_sizes) batch_sizes[count] = bs;
            if (ms_per_chunk) ms_per_chunk[count] = best;
        }
    }
    return count;
}

int select_batch_size(const int32_t* batch_sizes, const float* ms_per_chunk, int count, int max_batch_size, int granularity,
                      float time_penalty) {
    if (!batch_sizes || !ms_per_chunk || count < 1) throw std::invalid_argument("select_batch_size: empty table");
    if (!(time_penalty >= 0.0f)) throw std::invalid_argument("select_batch_size: negative time penalty");
    // entries that beat every smaller batch size, in ascending batch-size order
    std::vector<int> kept;
    float best = std::numeric_limits<float>::max();
    for (int i = 0; i < count; ++i) {
        if (i > 0 && batch_sizes[i] <= batch_sizes[i - 1]) throw std::invalid_argument("select_batch_size: batch sizes must ascend");
        if (ms_per_chunk[i] < best) {
            best = ms_per_chunk[i];
            kept.push_back(i);
        }
    }
    if (kept.empty()) throw std::invalid_argument("select_batch_size: no finite timing");
    const float threshold = best * (1.0f + time_penalty);
    size_t last = 0;
    while (last < kept.size() && !(ms_per_chunk[kept[last]] <= threshold)) ++last;  // first entry under the threshold
    int selected = granularity;
    for (size_t k = 0; k <= last && k < kept.size(); ++k) {
        if (batch_sizes[kept[k]] <= max_batch_size) selected = batch_sizes[kept[k]];
    }
    return selected;
}

void decode_host_scores(int device, const uint16_t* scores, int N, int T, int C, float clamp_val,
                        const b200_decoder_options& opts, uint8_t* moves, char* sequence, char* qstring,
                        int32_t* n_bases) {
    int state_len = 0;
    for (int sl = 3; sl <= 5; ++sl) {
        if (C == (1 << (2 * (sl + 1)))) state_len = sl;
    }
    if (!state_len) throw std::invalid_argument("decode: C must be 4^(state_len+1) with state_len 3..5");
    if (opts.move_pad != 0) throw Unsupported("move_pad: only the closed Koi kernel defines it; the reference never sets it");
    if (opts.temperature != 1.0f) throw Unsupported("temperature != 1: no decoder of the reference reads this option");
    require_sm90(device);
    cudaStream_t s;
    B200_CUDA(cudaStreamCreate(&s));
    size_t bwd_b = 0, beam_b = 0;
    decode_scratch_bytes(N, T, state_len, &bwd_b, &beam_b);
    const size_t sc_b = (size_t)N * T * C * sizeof(__half);
    const size_t out_b = nb_offset(N, T) + (size_t)N * 4;
    Arena arena;
    arena.reserve(sc_b + bwd_b + beam_b + out_b + 8192);
    auto* d_sc = static_cast<__half*>(arena.take(sc_b));
    b200_qtable tb;
    if (b200_qtable_build(opts.q_scale, opts.q_shift, &tb) != 0) {
        throw std::invalid_argument("decoder options: q_scale and q_shift must be finite");
    }
    auto* d_tb = static_cast<b200_qtable*>(arena.take(sizeof(b200_qtable)));
    DecodeArgs a{};
    a.scores = d_sc;
    a.N = N;
    a.T = T;
    a.state_len = state_len;
    a.clamp_val = clamp_val;
    a.beam_width = opts.beam_width;
    a.log_beam_cut = log_beam_cut_of(opts.beam_cut);
    a.blank = opts.blank_score;
    a.q_shift = opts.q_shift;
    a.q_scale = opts.q_scale;
    a.qtable = d_tb;
    a.bwd = static_cast<float*>(arena.take(bwd_b));
    a.beam = static_cast<uint2*>(arena.take(beam_b));
    auto* d_out = static_cast<unsigned char*>(arena.take(out_b));
    a.moves = d_out;
    a.sequence = reinterpret_cast<char*>(d_out + (size_t)N * T);
    a.qstring = reinterpret_cast<char*>(d_out + (size_t)2 * N * T);
    a.n_bases = reinterpret_cast<int32_t*>(d_out + nb_offset(N, T));
    try {
        B200_CUDA(cudaMemcpyAsync(d_sc, scores, sc_b, cudaMemcpyHostToDevice, s));
        B200_CUDA(cudaMemcpyAsync(d_tb, &tb, sizeof(tb), cudaMemcpyHostToDevice, s));
        long long* d_dbg = nullptr;
        if (std::getenv("B200_DEBUG_BEAM_TIMELINE")) {  // test hook only: clock64 stamps of chunk 0, blocks 100..107
            B200_CUDA(cudaMalloc(&d_dbg, 128 * sizeof(long long)));
            B200_CUDA(cudaMemsetAsync(d_dbg, 0, 128 * sizeof(long long), s));
            a.dbg = d_dbg;
        }
        decode_scores(a, s);
        if (std::getenv("B200_DEBUG_DECODE_TIMES")) {  // test hook only: per-kernel times of three more passes on the same scores
            for (int rep = 0; rep < 3; ++rep) {
                ProfileSink sink;
                sink.begin(s);
                decode_scores(a, s, &sink);
                B200_CUDA(cudaStreamSynchronize(s));
                std::string line = "[decode times]";
                for (auto& kv : sink.report()) line += " " + kv.first + "=" + std::to_string(kv.second);
                fprintf(stderr, "%s ms\n", line.c_str());
            }
        }
        if (d_dbg) {
            long long h[128];
            B200_CUDA(cudaMemcpyAsync(h, d_dbg, sizeof(h), cudaMemcpyDeviceToHost, s));
            B200_CUDA(cudaStreamSynchronize(s));
            for (int t = 0; t < 8; ++t) {
                const long long* e = h + t * 16;
                fprintf(stderr, "[beam timeline block %d] beam: wait %lld cand %lld merge %lld cutoff %lld compact %lld tail %lld (kept %lld) | "
                                "scan: wait_empty %lld work %lld | period %lld\n",
                        100 + t, e[0] - e[7], e[1] - e[0], e[2] - e[1], e[3] - e[2], e[4] - e[3], e[5] - e[4], e[6], e[9] - e[8],
                        e[10] - e[9], t > 0 ? e[0] - (e - 16)[0] : 0LL);
            }
            cudaFree(d_dbg);
        }
        B200_CUDA(cudaMemcpyAsync(moves, a.moves, (size_t)N * T, cudaMemcpyDeviceToHost, s));
        B200_CUDA(cudaMemcpyAsync(sequence, a.sequence, (size_t)N * T, cudaMemcpyDeviceToHost, s));
        B200_CUDA(cudaMemcpyAsync(qstring, a.qstring, (size_t)N * T, cudaMemcpyDeviceToHost, s));
        B200_CUDA(cudaMemcpyAsync(n_bases, a.n_bases, (size_t)N * 4, cudaMemcpyDeviceToHost, s));
        B200_CUDA(cudaStreamSynchronize(s));
    } catch (...) {
        cudaStreamDestroy(s);
        throw;
    }
    cudaStreamDestroy(s);
}

}  // namespace b200
