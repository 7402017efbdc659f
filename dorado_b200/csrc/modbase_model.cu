// Modified-base model conv_lstm_v3 for sm_90a: ModBaseConvLSTMV3Model::forward (dorado/modbase/nn/ModBaseModel.cpp:354-401),
// replacing the Koi path of ModBaseConvLSTMV3CUDAModel (:435-601).
//
//   signal encoder   sig_conv1 + sig_conv2     conv12_kernel (lstm_model.cu, FMA pipe) -> x2
//                    sig_conv3                 wgmma GEMM (gemm.cu), implicit im2col over x2, tanh/swish epilogue
//                                              -> merge input, channels [0, C_sig)
//   sequence encoder seq_conv1                 seq_conv1_kernel (FMA pipe, reads the int8 one-hot) -> y1
//                    seq_conv2                 wgmma GEMM, implicit im2col over y1 -> merge input, channels [C_sig, C_m)
//   merge_conv1                                wgmma GEMM, implicit im2col over the merge input -> sequence buffer
//   lstm1 (forward), lstm2 (reversed in time)  LstmStack (lstm_model.cu, the basecaller's LSTM stack)
//   linear, LinearUpsample, softmax            modbase_head_kernel -> fp16 [N][T_out][num_out]
//
// Implicit im2col: every convolution input is an NTC buffer whose rows are consecutive in memory, so the im2col row of
// output step t, the winlen input rows from stride * t on, is one contiguous run of winlen * C_in halves.  The GEMM's A
// operand reads it with a row stride of stride * C_in (overlapping rows), as conv3 of the basecaller does; zero rows
// before and after each chunk are the convolution's padding.  No im2col copy is materialised (0 extra bytes).
//
// Activation layouts in HBM (fp16), in workspace order:
//   seq       [T + 1][N][C]        LSTM sequence buffer: merge conv output, then h of each layer in place
//   x2        [N][Tp_sig][16]      sig_conv2 output, zero rows = sig_conv3's padding
//   y1        [N][Tp_seq][16]      seq_conv1 output, zero rows = seq_conv2's padding
//   merge_in  [N][Tp_m][C_m]       both encoders' outputs side by side, zero rows = the merge conv's padding
//   the LSTM stack's own slice (gx of the current layer, and the grid recurrence's counters and error word)
// The second LSTM runs reversed over the same time indices (the reference's flip, lstm, flip), so the sequence buffer is
// always in time order and the head reads it as it is.
#include "engine.h"
#include "gemm.h"
#include "lstm_kernels.h"
#include "nvtx.h"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>

namespace b200 {

namespace {

// ------------------------------------------------------------------------------------------------
// seq_conv1: int8 [N][T][C_in] (the k-mer one-hot as it arrives) -> fp16 [N][T_pad][16], stride 1, padding winlen / 2.
// One thread per output step, all 16 channels; the CTA's input window and the weights are staged in shared memory as
// fp32.  The reference casts the int8 to fp16 first (ModBaseModel.cpp:372-376): small integers convert exactly either way.
// ------------------------------------------------------------------------------------------------
constexpr int SQ_TT = 128;  // output steps per CTA

struct SeqConv1Params {
    const int8_t* x;  // [N][T][cin]
    __half* out;      // [N][T_pad][16], row r <-> step r - front_pad
    const float* w;   // [winlen][cin][16] | bias [16]
    int N, T, T_pad, front_pad, cin, winlen, act;
};

size_t seq_conv1_smem(int cin, int winlen) {
    return ((size_t)winlen * cin * 16 + 16 + (size_t)(SQ_TT + winlen - 1) * cin) * sizeof(float);
}
constexpr int SQ_MAX_SMEM = 227 * 1024;

__device__ __forceinline__ float mb_act(float v, int act) { return act == B200_ACT_TANH ? tanh_fast(v) : swish_fast(v); }

__global__ void __launch_bounds__(SQ_TT) seq_conv1_kernel(const SeqConv1Params p) {
    extern __shared__ __align__(16) float sq_smem[];
    const int nw = p.winlen * p.cin * 16;
    float* ws = sq_smem;                   // [winlen][cin][16], then the bias
    float* xs = sq_smem + nw + 16;         // [SQ_TT + winlen - 1][cin]
    const int n = blockIdx.y, t0 = blockIdx.x * SQ_TT, pad = p.winlen / 2;
    for (int i = threadIdx.x; i < nw + 16; i += SQ_TT) ws[i] = __ldg(p.w + i);
    const int rows = SQ_TT + p.winlen - 1;
    for (int i = threadIdx.x; i < rows * p.cin; i += SQ_TT) {
        const int t = t0 - pad + i / p.cin;
        xs[i] = (t >= 0 && t < p.T) ? (float)p.x[((size_t)n * p.T + t) * p.cin + i % p.cin] : 0.0f;
    }
    __syncthreads();
    const int t = t0 + threadIdx.x;
    if (t >= p.T) return;
    float acc[16];
#pragma unroll
    for (int co = 0; co < 16; ++co) acc[co] = ws[nw + co];
    for (int k = 0; k < p.winlen; ++k) {
        const float* xr = xs + (threadIdx.x + k) * p.cin;
        const float* wk = ws + k * p.cin * 16;
        for (int ci = 0; ci < p.cin; ++ci) {
            const float v = xr[ci];
            const float4* w4 = reinterpret_cast<const float4*>(wk + ci * 16);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float4 wv = w4[q];
                acc[4 * q + 0] = fmaf(v, wv.x, acc[4 * q + 0]);
                acc[4 * q + 1] = fmaf(v, wv.y, acc[4 * q + 1]);
                acc[4 * q + 2] = fmaf(v, wv.z, acc[4 * q + 2]);
                acc[4 * q + 3] = fmaf(v, wv.w, acc[4 * q + 3]);
            }
        }
    }
    __half2 h[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) h[j] = __floats2half2_rn(mb_act(acc[2 * j], p.act), mb_act(acc[2 * j + 1], p.act));
    uint4* dst = reinterpret_cast<uint4*>(p.out + ((size_t)n * p.T_pad + p.front_pad + t) * 16);
    dst[0] = *reinterpret_cast<const uint4*>(&h[0]);
    dst[1] = *reinterpret_cast<const uint4*>(&h[4]);
}

// ------------------------------------------------------------------------------------------------
// Head: linear (C -> num_out, + bias), optional LinearUpsample (num_out -> sf * num_out, + bias, reshaped to sf steps),
// softmax over the classes.  One warp per (t, chunk) row of the sequence buffer.  Rounded to fp16 where the reference's
// fp16 modules round: after the linear, after the upsample, after the softmax (its arithmetic is fp32).  The warp sum runs
// in a fixed butterfly order, so a chunk's result does not depend on its batch neighbours.
// ------------------------------------------------------------------------------------------------
constexpr int HEAD_WARPS = 8;
constexpr int HEAD_MAX_OUT = 10;  // MAX_FEATURES of ModBaseModelConfig.cpp:212
constexpr int HEAD_MAX_UP = 64;   // sf * num_out

struct HeadParams {
    const __half* seq;  // [T][N][C]
    const float* w;     // [num_out][C] (fp16 values)
    const float* b;     // [num_out] (fp16 values)
    const float* uw;    // [sf * num_out][num_out] (fp16 values), or null
    const float* ub;    // [sf * num_out] (fp16 values)
    __half* out;        // [N][T * sf][num_out]
    int T, N, C, num_out, sf;
};

__global__ void __launch_bounds__(HEAD_WARPS * 32) modbase_head_kernel(const HeadParams p) {
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * HEAD_WARPS + (threadIdx.x >> 5);  // row = t * N + n
    if (row >= p.T * p.N) return;
    const int t = row / p.N, n = row % p.N;
    const __half* x = p.seq + (size_t)row * p.C;
    float acc[HEAD_MAX_OUT];
#pragma unroll
    for (int o = 0; o < HEAD_MAX_OUT; ++o) acc[o] = 0.0f;
    for (int c8 = lane; c8 < p.C / 8; c8 += 32) {
        const uint4 raw = *reinterpret_cast<const uint4*>(x + c8 * 8);
        const __half2* hx = reinterpret_cast<const __half2*>(&raw);
        float xv[8];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 f = __half22float2(hx[j]);
            xv[2 * j] = f.x;
            xv[2 * j + 1] = f.y;
        }
#pragma unroll
        for (int o = 0; o < HEAD_MAX_OUT; ++o) {
            if (o < p.num_out) {
                const float4* w4 = reinterpret_cast<const float4*>(p.w + (size_t)o * p.C + c8 * 8);
                const float4 wa = __ldg(w4), wb = __ldg(w4 + 1);
                float a = acc[o];
                a = fmaf(xv[0], wa.x, a);
                a = fmaf(xv[1], wa.y, a);
                a = fmaf(xv[2], wa.z, a);
                a = fmaf(xv[3], wa.w, a);
                a = fmaf(xv[4], wb.x, a);
                a = fmaf(xv[5], wb.y, a);
                a = fmaf(xv[6], wb.z, a);
                a = fmaf(xv[7], wb.w, a);
                acc[o] = a;
            }
        }
    }
#pragma unroll
    for (int o = 0; o < HEAD_MAX_OUT; ++o) {
#pragma unroll
        for (int m = 16; m >= 1; m >>= 1) acc[o] += __shfl_xor_sync(0xffffffffu, acc[o], m);
    }
    // every lane holds the same sums; lane k < sf writes output step t * sf + k
    float y[HEAD_MAX_OUT];
#pragma unroll
    for (int o = 0; o < HEAD_MAX_OUT; ++o) y[o] = o < p.num_out ? __half2float(__float2half_rn(acc[o] + __ldg(p.b + o))) : 0.0f;
    const int steps = p.uw ? p.sf : 1;
    for (int k = lane; k < steps; k += 32) {
        float z[HEAD_MAX_OUT];
#pragma unroll
        for (int o = 0; o < HEAD_MAX_OUT; ++o) {
            z[o] = y[o];
            if (p.uw && o < p.num_out) {
                const int j = k * p.num_out + o;
                float a = 0.0f;
#pragma unroll
                for (int i = 0; i < HEAD_MAX_OUT; ++i) {
                    if (i < p.num_out) a = fmaf(y[i], __ldg(p.uw + (size_t)j * p.num_out + i), a);
                }
                z[o] = __half2float(__float2half_rn(a + __ldg(p.ub + j)));
            }
        }
        float mx = z[0];
#pragma unroll
        for (int o = 1; o < HEAD_MAX_OUT; ++o) mx = o < p.num_out ? fmaxf(mx, z[o]) : mx;
        float sum = 0.0f;
#pragma unroll
        for (int o = 0; o < HEAD_MAX_OUT; ++o) {
            z[o] = o < p.num_out ? expf(z[o] - mx) : 0.0f;
            sum += z[o];
        }
        const float inv = 1.0f / sum;
        __half* dst = p.out + ((size_t)n * p.T * steps + (size_t)t * steps + k) * p.num_out;
#pragma unroll
        for (int o = 0; o < HEAD_MAX_OUT; ++o) {
            if (o < p.num_out) dst[o] = __float2half_rn(z[o] * inv);
        }
    }
}

int conv_out_len(int len, const b200_conv_desc& c) { return (len + 2 * (c.winlen / 2) - c.winlen) / c.stride + 1; }
int round64(int k) { return (k + 63) / 64 * 64; }

}  // namespace

// ------------------------------------------------------------------------------------------------
// engine: weights in the kernels' layouts
// ------------------------------------------------------------------------------------------------
ModBaseEngine::ModBaseEngine(const b200_modbase_desc& d, const b200_tensor* tensors, int n, int device)
        : m_desc(d), m_device(device) {
    const auto &s1 = d.sig_convs[0], &s2 = d.sig_convs[1], &s3 = d.sig_convs[2];
    const auto &q1 = d.seq_convs[0], &q2 = d.seq_convs[1], &m = d.merge_conv;
    const b200_conv_desc* all[6] = {&s1, &s2, &s3, &q1, &q2, &m};
    for (const b200_conv_desc* c : all) {
        if (c->insize < 1 || c->size < 1 || c->winlen < 1 || c->stride < 1) throw std::invalid_argument("modbase: bad convolution shape");
        // ModsConv implements swish and tanh only (ModBaseModel.cpp:101-113)
        if (c->activation != B200_ACT_SWISH && c->activation != B200_ACT_TANH) throw std::invalid_argument("modbase: ModsConv has no fused clamp");
    }
    if (d.kmer_len < 1 || d.chunk_size < 1 || d.num_out < 1) throw std::invalid_argument("modbase: kmer_len, chunk_size and num_out must be positive");
    if (s2.insize != s1.size || s3.insize != s2.size || q1.insize != 4 * d.kmer_len || q2.insize != q1.size ||
        m.insize != s3.size + q2.size || m.size != d.lstm_size) {
        throw std::invalid_argument("modbase: convolution channel counts do not chain");
    }
    if (s1.insize != 1 || s1.stride != 1 || s2.stride != 1 || s1.size > 16 || s2.size != 16 || s1.winlen % 2 == 0 ||
        s2.winlen % 2 == 0 || s1.winlen > kConv12MaxWin || s2.winlen > kConv12MaxWin || q1.size != 16 || q1.stride != 1 ||
        q1.winlen % 2 == 0 || q2.stride != 1 || m.stride != 1 || s3.size % 32 != 0 || q2.size % 32 != 0) {
        throw Unsupported("modbase: convolution shapes outside what the kernels implement");
    }
    const int C = d.lstm_size;
    if (C != 128 && C != 192 && C != 256 && C != 384 && C != 768 && C != 1024) {
        throw Unsupported("modbase: lstm_size " + std::to_string(C) + " is not supported (128, 192, 256, 384, 768 and 1024 are)");
    }
    if (seq_conv1_smem(q1.insize, q1.winlen) > (size_t)SQ_MAX_SMEM) throw Unsupported("modbase: seq_conv1 too wide for shared memory");
    if (d.num_out > HEAD_MAX_OUT || d.upsample_scale < 0 || d.upsample_scale * d.num_out > HEAD_MAX_UP) {
        throw Unsupported("modbase: num_out / upsample scale outside what the head kernel implements");
    }
    // sequence input length: chunk_size / stride_ratio (ModBaseModelConfig.cpp:520-525); the sequence convs have stride 1
    const int sig_stride = s1.stride * s2.stride * s3.stride;
    if (d.chunk_size % sig_stride != 0) throw std::invalid_argument("modbase: chunk_size must be a multiple of the signal stride");
    sig_len = d.chunk_size;
    seq_len = d.chunk_size / sig_stride;
    t_enc = conv_out_len(conv_out_len(conv_out_len(sig_len, s1), s2), s3);
    if (conv_out_len(conv_out_len(seq_len, q1), q2) != t_enc) {
        throw std::invalid_argument("modbase: the signal and sequence encoders give different lengths");
    }
    T = conv_out_len(t_enc, m);
    if (T < 1) throw std::invalid_argument("modbase: chunk too short for the convolutions");
    out_len = T * std::max(1, d.upsample_scale);

    require_sm90(device);
    auto tensor = [&](const std::string& name, std::initializer_list<int64_t> dims) -> const float* {
        const b200_tensor& t = find_tensor(tensors, n, name);
        bool ok = t.data && t.ndim == (int)dims.size();
        int i = 0;
        for (int64_t v : dims) ok = ok && t.dims[i++] == v;
        if (!ok) throw std::invalid_argument("modbase: weight tensor '" + name + "' has the wrong shape");
        return t.data;
    };
    auto conv_tensors = [&](const std::string& name, const b200_conv_desc& c) {
        tensor(name + ".weight.tensor", {c.size, c.insize, c.winlen});
        tensor(name + ".bias.tensor", {c.size});
        return std::make_pair(&find_tensor(tensors, n, name + ".weight.tensor"), &find_tensor(tensors, n, name + ".bias.tensor"));
    };
    // GEMM weights of a convolution over NTC rows: [size][K padded to 64], K index = tap * insize + channel
    auto conv_gemm = [&](const std::string& name, const b200_conv_desc& c, __half** w, float** b) {
        const auto t = conv_tensors(name, c);
        const int K = round64(c.winlen * c.insize);
        std::vector<float> g((size_t)c.size * K, 0.0f);
        for (int co = 0; co < c.size; ++co)
            for (int ci = 0; ci < c.insize; ++ci)
                for (int k = 0; k < c.winlen; ++k)
                    g[(size_t)co * K + k * c.insize + ci] = t.first->data[((size_t)co * c.insize + ci) * c.winlen + k];
        *w = upload_f16(g);
        *b = upload_f32(std::vector<float>(t.second->data, t.second->data + c.size));
    };
    {
        const auto t1 = conv_tensors("sig_conv1", s1);
        const auto t2 = conv_tensors("sig_conv2", s2);
        sig12_w = upload_conv12_weights(*t1.first, *t1.second, *t2.first, *t2.second, s1, s2);
    }
    conv_gemm("sig_conv3", s3, &sig3_w, &sig3_b);
    {
        const auto t = conv_tensors("seq_conv1", q1);
        std::vector<float> w((size_t)q1.winlen * q1.insize * 16 + 16);
        for (int co = 0; co < 16; ++co) {
            for (int ci = 0; ci < q1.insize; ++ci)
                for (int k = 0; k < q1.winlen; ++k)
                    w[((size_t)k * q1.insize + ci) * 16 + co] = t.first->data[((size_t)co * q1.insize + ci) * q1.winlen + k];
            w[(size_t)q1.winlen * q1.insize * 16 + co] = t.second->data[co];
        }
        seq1_w = upload_f32(w);
    }
    conv_gemm("seq_conv2", q2, &seq2_w, &seq2_b);
    conv_gemm("merge_conv1", m, &merge_w, &merge_b);
    for (int l = 0; l < 2; ++l) {
        const std::string p = "lstm" + std::to_string(l + 1) + ".";
        lstm[l] = upload_lstm_layer(C, tensor(p + "weight_ih_l0.tensor", {4 * C, C}),
                                    tensor(p + "weight_hh_l0.tensor", {4 * C, C}), tensor(p + "bias_ih_l0.tensor", {4 * C}),
                                    tensor(p + "bias_hh_l0.tensor", {4 * C}));
    }
    // head: the reference's fp16 module holds fp16 weights and biases
    auto f16_values = [](const float* v, size_t count) {
        std::vector<float> out(count);
        for (size_t i = 0; i < count; ++i) out[i] = __half2float(__float2half_rn(v[i]));
        return out;
    };
    fc_w = upload_f32(f16_values(tensor("fc.weight.tensor", {d.num_out, C}), (size_t)d.num_out * C));
    fc_b = upload_f32(f16_values(tensor("fc.bias.tensor", {d.num_out}), (size_t)d.num_out));
    if (d.upsample_scale > 0) {
        const int U = d.upsample_scale * d.num_out;
        up_w = upload_f32(f16_values(tensor("linear_up.linear.weight.tensor", {U, d.num_out}), (size_t)U * d.num_out));
        up_b = upload_f32(f16_values(tensor("linear_up.linear.bias.tensor", {U}), (size_t)U));
    }
}

ModBaseEngine::~ModBaseEngine() {
    cudaSetDevice(m_device);
    for (void* p : {(void*)sig12_w, (void*)sig3_w, (void*)sig3_b, (void*)seq1_w, (void*)seq2_w, (void*)seq2_b, (void*)merge_w,
                    (void*)merge_b, (void*)fc_w, (void*)fc_b, (void*)up_w, (void*)up_b}) {
        cudaFree(p);
    }
    for (auto& l : lstm) free_lstm_layer(l);
}

// ------------------------------------------------------------------------------------------------
// runner: pinned batch, arena, launch plan
// ------------------------------------------------------------------------------------------------
struct ModBasePlan {
    Conv12Params sig12{};
    GemmPlan sig3, seq2, merge;
    SeqConv1Params seq1{};
    size_t seq1_smem = 0;
    std::unique_ptr<LstmStack> lstm;
    HeadParams head{};
};

ModBaseRunner::ModBaseRunner(ModBaseEngine& engine, int batch_size) : m_engine(engine), m_N(batch_size) {
    try {
        init();
    } catch (...) {
        release();
        throw;
    }
}

ModBaseRunner::~ModBaseRunner() { release(); }

void ModBaseRunner::release() {
    cudaSetDevice(m_engine.device());
    if (m_stream) cudaStreamSynchronize(m_stream);
    m_plan.reset();
    if (m_h_sig) cudaFreeHost(m_h_sig);
    if (m_h_kmers) cudaFreeHost(m_h_kmers);
    if (m_h_out) cudaFreeHost(m_h_out);
    m_h_sig = nullptr;
    m_h_kmers = nullptr;
    m_h_out = nullptr;
    if (m_stream) cudaStreamDestroy(m_stream);
    m_stream = nullptr;
}

void ModBaseRunner::init() {
    const ModBaseEngine& e = m_engine;
    const b200_modbase_desc& d = e.desc();
    const int N = m_N, C = d.lstm_size, T = e.T;
    // the LSTM recurrences take chunks in groups of 32 (the same rule as the basecaller's large LSTM sizes)
    if (N < 32 || N % 32 != 0) throw std::invalid_argument("modbase: batch_size must be a positive multiple of 32");
    const auto &s3 = d.sig_convs[2], &q1 = d.seq_convs[0], &q2 = d.seq_convs[1], &mc = d.merge_conv;
    m_kmer_elems = (int64_t)e.seq_len * q1.insize;
    m_out_elems = (int64_t)e.out_len * d.num_out;

    B200_CUDA(cudaSetDevice(e.device()));
    B200_CUDA(cudaStreamCreateWithFlags(&m_stream, cudaStreamNonBlocking));
    const size_t sig_b = (size_t)N * e.sig_len * 2, kmer_b = (size_t)N * m_kmer_elems, out_b = (size_t)N * m_out_elems * 2;
    B200_CUDA(cudaHostAlloc(&m_h_sig, sig_b, cudaHostAllocDefault));
    B200_CUDA(cudaHostAlloc(&m_h_kmers, kmer_b, cudaHostAllocDefault));
    B200_CUDA(cudaHostAlloc(&m_h_out, out_b, cudaHostAllocDefault));
    std::memset(m_h_sig, 0, sig_b);
    std::memset(m_h_kmers, 0, kmer_b);

    // padded row counts: each buffer holds the convolution's zero padding on both sides and enough rows after the last
    // window for the GEMM's K padding
    const int K3 = round64(s3.winlen * 16), K2 = round64(q2.winlen * 16), Km = round64(mc.winlen * mc.insize);
    const int Tp_sig = e.sig_len + 2 * (s3.winlen / 2) + K3 / 16;
    const int Tp_seq = e.seq_len + 2 * (q2.winlen / 2) + K2 / 16;
    const int Cm = mc.insize;
    const int Tp_m = e.t_enc + 2 * (mc.winlen / 2) + Km / Cm + 1;
    __half *seq = nullptr, *x2 = nullptr, *y1 = nullptr, *merge_in = nullptr;
    LstmStackBuffers lstm_ws;
    m_arena.allocate([&](Bump& b) {
        // the workspace: everything up to the input and output buffers
        seq = b.take<__half>((size_t)(T + 1) * N * C * 2);  // first: tests read it at offset 0
        x2 = b.take<__half>((size_t)N * Tp_sig * 16 * 2);
        y1 = b.take<__half>((size_t)N * Tp_seq * 16 * 2);
        merge_in = b.take<__half>((size_t)N * Tp_m * Cm * 2);
        lstm_ws = carve_lstm_stack(b, C, 2, T, N);
        m_ws_bytes = b.used();
        m_d_sig = b.take<__half>(sig_b);
        m_d_kmers = b.take<int8_t>(kmer_b);
        m_d_out = b.take<__half>(out_b);
    });
    m_d_ws = seq;
    // padding rows stay zero: the kernels write interior rows only
    B200_CUDA(cudaMemsetAsync(m_d_ws, 0, m_ws_bytes, m_stream));
    B200_CUDA(cudaMemsetAsync(m_d_sig, 0, sig_b, m_stream));
    B200_CUDA(cudaMemsetAsync(m_d_kmers, 0, kmer_b, m_stream));
    B200_CUDA(cudaStreamSynchronize(m_stream));

    auto plan = std::make_unique<ModBasePlan>();
    const auto &s1 = d.sig_convs[0], &s2 = d.sig_convs[1];
    plan->sig12 = Conv12Params{m_d_sig, x2, e.sig12_w, N, e.sig_len, Tp_sig, s3.winlen / 2, s1.size, s1.winlen, s2.winlen,
                               s1.activation, s2.activation, nullptr, nullptr};
    plan->seq1 = SeqConv1Params{m_d_kmers, y1, e.seq1_w, N, e.seq_len, Tp_seq, q2.winlen / 2, q1.insize, q1.winlen, q1.activation};
    plan->seq1_smem = seq_conv1_smem(q1.insize, q1.winlen);
    // the attribute is set once per device for every model the process loads: the largest size the engine accepts
    ensure_dynamic_smem(seq_conv1_kernel, SQ_MAX_SMEM);
    // encoder convolutions: rows (chunk, t) of the input NTC buffer, written into the merge input at row padm + t
    const int padm = mc.winlen / 2;
    auto encoder_gemm = [&](const __half* a, int Tp, int stride, int K, const __half* w, const float* b, int cols,
                            int act, int col0) {
        GemmDesc g{};
        g.a = a;
        g.batches = N;
        g.rows_per_batch = e.t_enc;
        g.a_row_stride = (int64_t)stride * 16;
        g.a_batch_stride = (int64_t)Tp * 16;
        g.w = w;
        g.N = cols;
        g.K = K;
        g.bias = b;
        g.act = act;
        g.out = merge_in + (size_t)padm * Cm + col0;
        g.out_m1 = e.t_enc;                 // g = n * t_enc + t
        g.out_s0 = (int64_t)Tp_m * Cm;      // n
        g.out_s1 = Cm;                      // t
        return make_gemm_plan(g);
    };
    plan->sig3 = encoder_gemm(x2, Tp_sig, s3.stride, K3, e.sig3_w, e.sig3_b, s3.size, s3.activation, 0);
    plan->seq2 = encoder_gemm(y1, Tp_seq, 1, K2, e.seq2_w, e.seq2_b, q2.size, q2.activation, s3.size);
    {
        GemmDesc g{};
        g.a = merge_in;
        g.batches = N;
        g.rows_per_batch = T;
        g.a_row_stride = Cm;
        g.a_batch_stride = (int64_t)Tp_m * Cm;
        g.w = e.merge_w;
        g.N = C;
        g.K = Km;
        g.bias = e.merge_b;
        g.act = mc.activation;
        g.out = seq;
        g.out_m1 = T;                   // g = n * T + t
        g.out_s0 = C;                   // n
        g.out_s1 = (int64_t)N * C;      // t
        plan->merge = make_gemm_plan(g);
    }
    // sized for dorado's default of two runners per device (api/runner_creation.cpp:46-130); lstm1 runs forward in time,
    // lstm2 over the flipped sequence (ModBaseModel.cpp:384-392)
    LstmStackDesc lstm{};
    lstm.C = C;
    lstm.T = T;
    lstm.Np = N;
    lstm.runners = 2;
    lstm.seq = seq;
    lstm.layers = e.lstm;
    lstm.num_layers = 2;
    plan->lstm = std::make_unique<LstmStack>(lstm, lstm_ws);
    plan->head = HeadParams{seq, e.fc_w, e.fc_b, e.up_w, e.up_b, m_d_out, T, N, C, d.num_out, std::max(1, d.upsample_scale)};
    m_plan = std::move(plan);
}

void ModBaseRunner::accept_chunk(int idx, const uint16_t* signal, int64_t sig_len, const int8_t* kmers, int64_t kmer_elems) {
    if (idx < 0 || idx >= m_N) throw std::invalid_argument("modbase accept_chunk: chunk index out of range");
    if (!signal || !kmers) throw std::invalid_argument("modbase accept_chunk: null input");
    // the reference throws std::logic_error on a signal of another length (ModBaseRunner.cpp:57-60)
    if (sig_len != m_engine.sig_len) {
        throw std::invalid_argument("modbase accept_chunk: signal of " + std::to_string(sig_len) + " samples, the model takes " +
                                    std::to_string(m_engine.sig_len));
    }
    if (kmer_elems != m_kmer_elems) {
        throw std::invalid_argument("modbase accept_chunk: " + std::to_string(kmer_elems) + " k-mer values, the model takes " +
                                    std::to_string(m_kmer_elems));
    }
    std::memcpy(m_h_sig + (size_t)idx * sig_len, signal, (size_t)sig_len * 2);
    std::memcpy(m_h_kmers + (size_t)idx * kmer_elems, kmers, (size_t)kmer_elems);
}

void ModBaseRunner::run(ProfileSink* prof) {
    ModBasePlan& p = *m_plan;
    cudaStream_t s = m_stream;
    auto mark = [&](const char* name) {
        if (prof) prof->mark(name, s);
    };
    {
        NvtxRange r("modbase_encoders");
        launch_conv12(p.sig12, s);
        mark("sig_conv12");
        run_gemm(p.sig3, s);
        mark("sig_conv3_gemm");
        seq_conv1_kernel<<<dim3((p.seq1.T + SQ_TT - 1) / SQ_TT, p.seq1.N, 1), SQ_TT, p.seq1_smem, s>>>(p.seq1);
        mark("seq_conv1");
        run_gemm(p.seq2, s);
        mark("seq_conv2_gemm");
        run_gemm(p.merge, s);
        mark("merge_conv_gemm");
    }
    if (!p.lstm->run(s, prof)) {  // debug: the sequence buffer holds the output of B200_DEBUG_LSTM_LAYERS layers
        B200_CUDA(cudaGetLastError());
        return;
    }
    NvtxRange r("modbase_head");
    const int rows = p.head.T * p.head.N;
    modbase_head_kernel<<<(rows + HEAD_WARPS - 1) / HEAD_WARPS, HEAD_WARPS * 32, 0, s>>>(p.head);
    mark("head");
    B200_CUDA(cudaGetLastError());
}

const uint16_t* ModBaseRunner::call_chunks(int num_chunks) {
    if (num_chunks < 1 || num_chunks > m_N) throw std::invalid_argument("modbase call_chunks: num_chunks out of range");
    std::lock_guard<std::mutex> lock(m_mutex);
    B200_CUDA(cudaSetDevice(m_engine.device()));
    cudaStream_t s = m_stream;
    const int sig_len = m_engine.sig_len;
    B200_CUDA(cudaMemcpyAsync(m_d_sig, m_h_sig, (size_t)num_chunks * sig_len * 2, cudaMemcpyHostToDevice, s));
    B200_CUDA(cudaMemcpyAsync(m_d_kmers, m_h_kmers, (size_t)num_chunks * m_kmer_elems, cudaMemcpyHostToDevice, s));
    run(nullptr);
    B200_CUDA(cudaMemcpyAsync(m_h_out, m_d_out, (size_t)num_chunks * m_out_elems * 2, cudaMemcpyDeviceToHost, s));
    B200_CUDA(cudaStreamSynchronize(s));
    m_plan->lstm->check_errors();
    return reinterpret_cast<const uint16_t*>(m_h_out);
}

std::string ModBaseRunner::profile() {
    std::lock_guard<std::mutex> lock(m_mutex);
    B200_CUDA(cudaSetDevice(m_engine.device()));
    ProfileSink sink;
    sink.begin(m_stream);
    run(&sink);
    B200_CUDA(cudaStreamSynchronize(m_stream));
    m_plan->lstm->check_errors();
    std::string out;
    for (auto& kv : sink.report()) out += kv.first + "=" + std::to_string(kv.second) + ";";
    return out;
}

void ModBaseRunner::debug_read_workspace(uint64_t offset, uint64_t bytes, void* dst) {
    if (offset > m_ws_bytes || bytes > m_ws_bytes - offset) throw std::invalid_argument("debug_read_workspace: out of range");
    std::lock_guard<std::mutex> lock(m_mutex);
    B200_CUDA(cudaSetDevice(m_engine.device()));
    B200_CUDA(cudaStreamSynchronize(m_stream));
    B200_CUDA(cudaMemcpy(dst, static_cast<unsigned char*>(m_d_ws) + offset, bytes, cudaMemcpyDeviceToHost));
}

}  // namespace b200
