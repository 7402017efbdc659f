// Conv -> Transformer encoder -> upsample -> scaled CRF linear forward (sup models) for sm_90a.
//
// Replaces the CUDA path of dorado/basecall/model/TxModel.cpp:20-41 and dorado/nn/TxModules.cpp:
//   conv stack (torch conv1d on the reference's CUDA path)   ConvStack.cpp:146-163    -> conv1 kernel + gemm.cu
//   koi_qkv_rotary / koi_masked_attention                    TxModules.cpp:642-648    -> gemm.cu + tx_attention_tc_kernel
//   koi_linear (out_proj, fc2) + koi_rmsnorm_residual        TxModules.cpp:653-712    -> gemm.cu (fused residual) + rmsnorm
//   koi_mm_swiglu                                            TxModules.cpp:683        -> gemm.cu (SwiGLU epilogue)
//   LinearUpsample, LinearScaledCRF                          LinearUpsample.cpp:17-23, TxModules.cpp:1010-1016 -> gemm.cu
// Semantics follow the CPU modules: TxEncoderImpl::forward (TxModules.cpp:859-906), MultiHeadAttentionImpl
// (:346-426, true window -win_upper <= j - i <= win_lower, see oracle/nn_oracle.py on the CPU split quirk), RotaryEmbedding
// (:220-250, half-split rotation), GatedMLP (:170-176), RMSNorm (RMSNorm.cpp:14-18).
//
// Activations are NTC fp16.  Every conv after the first is a strided GEMM over the zero-padded NTC buffer of
// the previous layer (row stride = stride * C_in), all projections are wgmma GEMMs; the residual stream is
// x <- RMSNorm(sublayer(x) + alpha * x) with the "+ alpha * x" fused into the GEMM epilogue.
#include "engine.h"
#include "gemm.h"
#include "nvtx.h"

#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>

namespace b200 {

namespace {

__device__ __forceinline__ float swish_f(float v) { return swish_fast(v); }

// ------------------------------------------------------------------------------------------------
// conv1: 1 -> C1 channels, stride 1.  out[n][pad_out + t][c] = swish(b[c] + sum_k w[c][k] x[n][t + k - W/2])
// ------------------------------------------------------------------------------------------------
struct Conv1Params {
    const __half* x;   // [N][T]
    __half* out;       // [N][T_pad][C1]
    const float* w;    // [C1][W] then bias [C1]
    int N, T, T_pad, pad_out, C1, W, act;
};

__global__ void __launch_bounds__(256) tx_conv1_kernel(const Conv1Params p) {
    // thread = (t, group of 8 channels)
    const int groups = p.C1 / 8;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)p.N * p.T * groups;
    if (idx >= total) return;
    const int cg = (int)(idx % groups);
    const long long nt = idx / groups;
    const int t = (int)(nt % p.T);
    const int n = (int)(nt / p.T);
    float xs[9];
    const int half_w = p.W / 2;
    for (int k = 0; k < p.W; ++k) {
        const int tt = t + k - half_w;
        xs[k] = (tt >= 0 && tt < p.T) ? __half2float(p.x[(size_t)n * p.T + tt]) : 0.0f;
    }
    __half2 h[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        float v[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int c = cg * 8 + 2 * j + e;
            float acc = __ldg(p.w + p.C1 * p.W + c);
            for (int k = 0; k < p.W; ++k) acc += __ldg(p.w + c * p.W + k) * xs[k];
            v[e] = p.act == B200_ACT_TANH ? tanh_fast(acc)
                                          : (p.act == B200_ACT_SWISH_CLAMP ? fminf(swish_f(acc), 3.5f) : swish_f(acc));
        }
        h[j] = __floats2half2_rn(v[0], v[1]);
    }
    *reinterpret_cast<uint4*>(p.out + ((size_t)n * p.T_pad + p.pad_out + t) * p.C1 + cg * 8) = *reinterpret_cast<uint4*>(h);
}

// ------------------------------------------------------------------------------------------------
// RMSNorm over rows of 512 (RMSNorm.cpp:14-18): x * rsqrt(mean(x^2) + eps) * w ; one warp per row.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) rmsnorm512_kernel(const __half* __restrict__ in, __half* __restrict__ out,
                                                         const float* __restrict__ w, long long rows) {
    const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const uint4* src = reinterpret_cast<const uint4*>(in + row * 512) + lane * 2;
    uint4 v[2] = {src[0], src[1]};
    float f[16];
    float ss = 0.0f;
#pragma unroll
    for (int q = 0; q < 2; ++q) {
        const __half2* h = reinterpret_cast<const __half2*>(&v[q]);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 a = __half22float2(h[j]);
            f[q * 8 + 2 * j] = a.x;
            f[q * 8 + 2 * j + 1] = a.y;
            ss += a.x * a.x + a.y * a.y;
        }
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float rstd = rsqrtf(ss * (1.0f / 512.0f) + 1e-5f);
    __half2 o2[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int c = lane * 16 + 2 * j;
        o2[j] = __floats2half2_rn(f[2 * j] * rstd * __ldg(w + c), f[2 * j + 1] * rstd * __ldg(w + c + 1));
    }
    uint4* dst = reinterpret_cast<uint4*>(out + row * 512) + lane * 2;
    dst[0] = *reinterpret_cast<uint4*>(&o2[0]);
    dst[1] = *reinterpret_cast<uint4*>(&o2[4]);
}

constexpr int ATT_D = 64;   // head dimension

// ------------------------------------------------------------------------------------------------
// Sliding-window attention on the tensor cores (successor of koi_masked_attention, TxModules.cpp:648; window semantics
// TxModules.cpp:310-317: keys j with -win_upper <= j - i <= win_lower).
// qkv: [N*T][3][H][64] fp16 (output of the Wqkv GEMM, q and k already rotated); out: [N*T][H*64] fp16.
// One CTA = 128 queries of one (chunk, head); the keys they can see lie in at most three aligned blocks of 128 keys (the
// kernel requires win_upper + win_lower + 128 <= 3 * 128).  One thread loads Q and every K / V block up front by TMA
// (128-byte swizzle); each of the eight warps then owns 16 query rows and walks the blocks flash-style on mma.sync:
//     S_b = Q K_b^T          16 x 128 per warp, fp32 in registers (Q and K_b fragments by ldmatrix)
//     P_b = exp2(S_b' - m)   running max / sum per row (the four lanes of a quad share a row), P rounded to fp16 and
//                            re-used in registers as the A fragments of the next product
//     O = O * alpha + P_b V_b  V_b as it lies in memory ([key][d]) through ldmatrix.trans -- no transposed copy of V
// Shared memory 113 KB: two CTAs share an SM.
// ------------------------------------------------------------------------------------------------
constexpr int AT_BQ = 128, AT_BK = 128;
constexpr int AT_TILE = 128 * 64 * 2;   // one [128 x 64] fp16 tile
constexpr int AT_MAXBLK = 3;
constexpr int AT_THREADS = 256;
constexpr int AT_SMEM = 1024 + (1 + 2 * AT_MAXBLK) * AT_TILE + 64;

struct AttnTcParams {
    __half* out;   // [N*T][H*64]
    int N, T, H;
    int win_upper, win_lower;
};

__global__ void __launch_bounds__(AT_THREADS, 2) tx_attention_tc_kernel(const __grid_constant__ CUtensorMap tma_qkv, const AttnTcParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* q_s = smem;                          // [128 q][64 d]
    uint8_t* k_s = q_s + AT_TILE;                 // [3][128 keys][64 d]
    uint8_t* v_s = k_s + AT_MAXBLK * AT_TILE;     // [3][128 keys][64 d]
    uint64_t* bars = reinterpret_cast<uint64_t*>(v_s + AT_MAXBLK * AT_TILE);
    uint64_t* q_full = bars;          // TMA -> warps
    uint64_t* kv_full = bars + 1;     // [3]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int qt = blockIdx.x, h = blockIdx.y, n = blockIdx.z;
    const int q0 = qt * AT_BQ;
    // aligned key blocks that intersect [q0 - win_upper, q0 + 127 + win_lower] and [0, T)
    int kb_first = (q0 - p.win_upper) / AT_BK;   // q0 >= 0, so this only goes negative through the subtraction
    if (q0 - p.win_upper < 0) kb_first = 0;
    int kb_last = (q0 + AT_BQ - 1 + p.win_lower) / AT_BK;
    const int kb_max = (p.T - 1) / AT_BK;
    if (kb_last > kb_max) kb_last = kb_max;
    const int nblk = kb_last - kb_first + 1;     // 1..3 (checked on the host)
    const int row0 = n * p.T;   // first token row of this chunk in the [N*T][1536] view

    if (threadIdx.x == 0) {
        tc::mbar_init(q_full, 1);
        for (int i = 0; i < AT_MAXBLK; ++i) tc::mbar_init(&kv_full[i], 1);
        tc::fence_barrier_init();
        tc::prefetch_tmap(&tma_qkv);
        tc::mbar_arrive_expect_tx(q_full, AT_TILE);
        tc::tma_load_2d(q_s, &tma_qkv, q_full, h * ATT_D, row0 + q0);
        for (int b = 0; b < nblk; ++b) {
            tc::mbar_arrive_expect_tx(&kv_full[b], 2 * AT_TILE);
            const int krow = row0 + (kb_first + b) * AT_BK;
            tc::tma_load_2d(k_s + b * AT_TILE, &tma_qkv, &kv_full[b], (p.H + h) * ATT_D, krow);
            tc::tma_load_2d(v_s + b * AT_TILE, &tma_qkv, &kv_full[b], (2 * p.H + h) * ATT_D, krow);
        }
    }
    __syncthreads();

    const int qm = lane >> 3, qr = lane & 7;   // ldmatrix.x4: matrix qm, row qr
    const int quad = lane & 3;
    const float sc = 0.125f * 1.44269504088896341f;   // 1/sqrt(64) and the base change of exp -> exp2
    int qi[2];
    qi[0] = q0 + warp * 16 + (lane >> 2);
    qi[1] = qi[0] + 8;
    tc::mbar_wait(q_full, 0);
    uint32_t qa[ATT_D / 16][4];   // A fragments of this warp's 16 query rows; matrix qm = (row half qm % 2, d half qm / 2)
#pragma unroll
    for (int ks = 0; ks < ATT_D / 16; ++ks) {
        tc::ldmatrix_x4(qa[ks], tc::smem_u32(q_s + tc::sw128_offset(warp * 16 + (qm & 1) * 8 + qr, 2 * ks + (qm >> 1))));
    }
    float o[ATT_D / 8][4];
#pragma unroll
    for (int dt = 0; dt < ATT_D / 8; ++dt) o[dt][0] = o[dt][1] = o[dt][2] = o[dt][3] = 0.0f;
    float m_run[2] = {-1e30f, -1e30f}, l_run[2] = {0.0f, 0.0f};

    for (int b = 0; b < nblk; ++b) {
        const int kb = (kb_first + b) * AT_BK;
        const uint8_t* kt = k_s + b * AT_TILE;
        const uint8_t* vt = v_s + b * AT_TILE;
        // keys of this block visible to each row: j in [lo, hi)
        int lo[2], hi[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            lo[r] = max(qi[r] - p.win_upper - kb, 0);
            hi[r] = min(min(qi[r] + p.win_lower + 1 - kb, AT_BK), p.T - kb);
            if (qi[r] >= p.T) hi[r] = 0;
        }
        tc::mbar_wait(&kv_full[b], 0);
        // S = Q K^T: 16 key tiles of 8; K fragments: matrix qm = (key tile 2 np + qm / 2, d half qm % 2)
        float sacc[AT_BK / 8][4];
#pragma unroll
        for (int nt = 0; nt < AT_BK / 8; ++nt) sacc[nt][0] = sacc[nt][1] = sacc[nt][2] = sacc[nt][3] = 0.0f;
#pragma unroll
        for (int ks = 0; ks < ATT_D / 16; ++ks) {
#pragma unroll
            for (int np = 0; np < AT_BK / 16; ++np) {
                uint32_t kf[4];
                tc::ldmatrix_x4(kf, tc::smem_u32(kt + tc::sw128_offset((2 * np + (qm >> 1)) * 8 + qr, 2 * ks + (qm & 1))));
                tc::mma_f16_16816(sacc[2 * np], qa[ks], kf[0], kf[1]);
                tc::mma_f16_16816(sacc[2 * np + 1], qa[ks], kf[2], kf[3]);
            }
        }
        // masked row maxima (a row's 128 keys are spread over the four lanes of its quad)
        float m_blk[2] = {-1e30f, -1e30f};
#pragma unroll
        for (int nt = 0; nt < AT_BK / 8; ++nt) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int r = e >> 1, j = nt * 8 + 2 * quad + (e & 1);
                if (j >= lo[r] && j < hi[r]) m_blk[r] = fmaxf(m_blk[r], sacc[nt][e]);
            }
        }
        float alpha[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            m_blk[r] = fmaxf(m_blk[r], __shfl_xor_sync(0xffffffffu, m_blk[r], 1));
            m_blk[r] = fmaxf(m_blk[r], __shfl_xor_sync(0xffffffffu, m_blk[r], 2));
            const float m_new = fmaxf(m_run[r], m_blk[r] * sc);
            alpha[r] = ex2_approx(m_run[r] - m_new);   // 1 when nothing changed, 0 on the first visible block
            m_run[r] = m_new;
            l_run[r] *= alpha[r];
        }
#pragma unroll
        for (int dt = 0; dt < ATT_D / 8; ++dt) {
            o[dt][0] *= alpha[0]; o[dt][1] *= alpha[0];
            o[dt][2] *= alpha[1]; o[dt][3] *= alpha[1];
        }
        // P = exp2(S * sc - m), then O += P V one 16-key step at a time: P's C fragments of key tiles 2 kk, 2 kk + 1 are
        // the A fragment of the step; V fragments by ldmatrix.trans, matrix qm = (key half qm % 2, d tile 2 dp + qm / 2)
#pragma unroll
        for (int kk = 0; kk < AT_BK / 16; ++kk) {
            float pv[2][4];
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int nt = 2 * kk + i;
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int r = e >> 1, j = nt * 8 + 2 * quad + (e & 1);
                    pv[i][e] = (j >= lo[r] && j < hi[r]) ? ex2_approx(fmaf(sacc[nt][e], sc, -m_run[r])) : 0.0f;
                }
                l_run[0] += pv[i][0] + pv[i][1];
                l_run[1] += pv[i][2] + pv[i][3];
            }
            uint32_t pa[4];
            pa[0] = tc::pack_half2(pv[0][0], pv[0][1]);
            pa[1] = tc::pack_half2(pv[0][2], pv[0][3]);
            pa[2] = tc::pack_half2(pv[1][0], pv[1][1]);
            pa[3] = tc::pack_half2(pv[1][2], pv[1][3]);
#pragma unroll
            for (int dp = 0; dp < ATT_D / 16; ++dp) {
                uint32_t vf[4];
                tc::ldmatrix_x4_trans(vf, tc::smem_u32(vt + tc::sw128_offset(16 * kk + (qm & 1) * 8 + qr, 2 * dp + (qm >> 1))));
                tc::mma_f16_16816(o[2 * dp], pa, vf[0], vf[1]);
                tc::mma_f16_16816(o[2 * dp + 1], pa, vf[2], vf[3]);
            }
        }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
        l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
        if (qi[r] >= p.T) continue;
        const float inv = l_run[r] > 0.0f ? 1.0f / l_run[r] : 0.0f;
        __half* dst = p.out + ((size_t)row0 + qi[r]) * (size_t)(p.H * ATT_D) + (size_t)h * ATT_D + 2 * quad;
#pragma unroll
        for (int dt = 0; dt < ATT_D / 8; ++dt) {
            *reinterpret_cast<__half2*>(dst + dt * 8) = __floats2half2_rn(o[dt][2 * r] * inv, o[dt][2 * r + 1] * inv);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
struct TxLayerWeights {
    __half *wqkv = nullptr, *wo = nullptr, *w1 = nullptr, *w2 = nullptr;
    float *bo = nullptr, *n1 = nullptr, *n2 = nullptr;
};

class TxModel;

class TxPlan final : public ForwardPlan {
public:
    void run(cudaStream_t stream, ProfileSink* prof) override;
    int launches() const override { return n_launches; }
    Conv1Params conv1{};
    std::vector<GemmPlan> convs;  // conv 2..n
    struct Layer {
        GemmPlan qkv, out_proj, fc1, fc2;
        const float *n1, *n2;
    };
    std::vector<Layer> layers;
    GemmPlan upsample, crf;
    CUtensorMap qkv_map;       // qkv as [N*T][3*H*64], box 64 x 128 (Q, K and V tiles of the tensor-core attention)
    AttnTcParams attn_tc_p{};
    __half *x = nullptr, *y = nullptr;
    long long rows = 0;
    int N = 0, T = 0, H = 0;
    int n_launches = 0;
    bool fold_norm = true;
};

class TxModel final : public Model {
public:
    TxModel(const b200_model_desc& d, const b200_tensor* tensors, int n);
    ~TxModel() override;
    size_t workspace_bytes(int N, int T_in) const override;
    std::unique_ptr<ForwardPlan> make_plan(int N, int T_in, const __half* signal, __half* scores, void* ws,
                                           size_t ws_bytes) override;
    b200_model_desc desc;
    bool fold_norm = true;   // B200_TX_RMSNORM_PASS=1: separate RMSNorm kernel after every sub-layer (A/B comparisons)
    float* conv1_w = nullptr;
    std::vector<__half*> conv_w;  // conv 2..n  [C_out][W*C_in]
    std::vector<float*> conv_b;
    std::vector<TxLayerWeights> layers;
    __half *wu = nullptr, *wc = nullptr;
    float* bu = nullptr;
    float* rope = nullptr;
    std::vector<void*> owned;

private:
    struct Shapes {
        std::vector<int> t;      // time length after conv i
        std::vector<int> t_pad;  // padded rows of the buffer holding conv i's output
        std::vector<int> pad;    // front padding of that buffer (= next conv's winlen/2)
    };
    Shapes shapes(int T_in) const;
};

TxModel::Shapes TxModel::shapes(int T_in) const {
    Shapes s;
    int t = T_in;
    for (int i = 0; i < desc.num_convs; ++i) {
        const auto& c = desc.convs[i];
        t = (t + 2 * (c.winlen / 2) - c.winlen) / c.stride + 1;
        const int next_pad = i + 1 < desc.num_convs ? desc.convs[i + 1].winlen / 2 : 0;
        s.t.push_back(t);
        s.pad.push_back(next_pad);
        s.t_pad.push_back(t + 2 * next_pad + 16);
    }
    return s;
}

TxModel::TxModel(const b200_model_desc& d, const b200_tensor* tensors, int n) : desc(d) {
    if (const char* e = std::getenv("B200_TX_RMSNORM_PASS")) fold_norm = std::atoi(e) == 0;
    if (d.d_model != 512 || d.nhead != 8) throw Unsupported("transformer path implements d_model 512, 8 heads (sup)");
    if (d.num_convs < 2 || d.convs[0].insize != 1 || d.convs[0].stride != 1 || d.convs[0].winlen > 9 || d.convs[0].size % 8) {
        throw Unsupported("transformer conv stack shape not supported");
    }
    if (d.convs[d.num_convs - 1].size != d.d_model) throw std::invalid_argument("last conv size != d_model");
    auto up16 = [&](const std::vector<float>& v) {
        __half* p = upload_f16(v);
        owned.push_back(p);
        return p;
    };
    auto up32 = [&](const float* data, size_t cnt) {
        float* p = upload_f32(std::vector<float>(data, data + cnt));
        owned.push_back(p);
        return p;
    };
    {
        const auto& tw = find_tensor(tensors, n, "conv.0.conv.weight.tensor");
        const auto& tb = find_tensor(tensors, n, "conv.0.conv.bias.tensor");
        const int c1 = d.convs[0].size, w = d.convs[0].winlen;
        std::vector<float> pk((size_t)c1 * w + c1);
        std::memcpy(pk.data(), tw.data, sizeof(float) * (size_t)c1 * w);
        std::memcpy(pk.data() + (size_t)c1 * w, tb.data, sizeof(float) * c1);
        conv1_w = up32(pk.data(), pk.size());
    }
    for (int i = 1; i < d.num_convs; ++i) {
        const auto& c = d.convs[i];
        const std::string pfx = "conv." + std::to_string(i) + ".conv.";
        const auto& tw = find_tensor(tensors, n, pfx + "weight.tensor");
        const auto& tb = find_tensor(tensors, n, pfx + "bias.tensor");
        const int K = c.winlen * c.insize;
        if (K % 64 != 0 || c.size % 32 != 0) throw Unsupported("conv K = winlen * insize must be a multiple of 64");
        std::vector<float> w((size_t)c.size * K);
        for (int co = 0; co < c.size; ++co)
            for (int ci = 0; ci < c.insize; ++ci)
                for (int k = 0; k < c.winlen; ++k)
                    w[(size_t)co * K + (size_t)k * c.insize + ci] = tw.data[((size_t)co * c.insize + ci) * c.winlen + k];
        conv_w.push_back(up16(w));
        conv_b.push_back(up32(tb.data, c.size));
    }
    const int dm = d.d_model, ff = d.dim_feedforward;
    // RMSNorm is folded into the GEMMs around it (gemm.h): x' = u * rsqrt(mean(u^2) + eps) * gain is never materialised.  The
    // consumers of x' scale their accumulator rows by 1/rms and have the gain folded into their weight COLUMNS here.
    auto fold = [&](const float* w, size_t rows, const float* gain) {
        std::vector<float> out(rows * (size_t)dm);
        for (size_t r = 0; r < rows; ++r)
            for (int c = 0; c < dm; ++c) out[r * dm + c] = w[r * dm + c] * (gain ? gain[c] : 1.0f);
        return out;
    };
    const float* prev_gain = nullptr;   // norm2 gain of the previous layer (none before layer 0: the conv output is used as is)
    for (int l = 0; l < d.depth; ++l) {
        const std::string pfx = "transformer_encoder." + std::to_string(l) + ".";
        TxLayerWeights lw;
        const float* n1 = find_tensor(tensors, n, pfx + "norm1.weight.tensor").data;
        const float* n2 = find_tensor(tensors, n, pfx + "norm2.weight.tensor").data;
        const auto& wqkv = find_tensor(tensors, n, pfx + "self_attn.Wqkv.weight.tensor");
        lw.wqkv = up16(fold_norm ? fold(wqkv.data, (size_t)3 * dm, prev_gain) : std::vector<float>(wqkv.data, wqkv.data + (size_t)3 * dm * dm));
        const auto& wo = find_tensor(tensors, n, pfx + "self_attn.out_proj.weight.tensor");
        lw.wo = up16(std::vector<float>(wo.data, wo.data + (size_t)dm * dm));
        lw.bo = up32(find_tensor(tensors, n, pfx + "self_attn.out_proj.bias.tensor").data, dm);
        // fc1 rows [y(0..ff) | gate(0..ff)] (TxModules.cpp:170-176) interleaved to (y_j, gate_j) pairs
        const auto& w1 = find_tensor(tensors, n, pfx + "ff.fc1.weight.tensor");
        std::vector<float> w1i((size_t)2 * ff * dm);
        for (int j = 0; j < ff; ++j) {
            std::memcpy(&w1i[(size_t)(2 * j) * dm], &w1.data[(size_t)j * dm], sizeof(float) * dm);
            std::memcpy(&w1i[(size_t)(2 * j + 1) * dm], &w1.data[(size_t)(ff + j) * dm], sizeof(float) * dm);
        }
        lw.w1 = up16(fold_norm ? fold(w1i.data(), (size_t)2 * ff, n1) : w1i);
        prev_gain = n2;
        const auto& w2 = find_tensor(tensors, n, pfx + "ff.fc2.weight.tensor");
        lw.w2 = up16(std::vector<float>(w2.data, w2.data + (size_t)dm * ff));
        lw.n1 = up32(find_tensor(tensors, n, pfx + "norm1.weight.tensor").data, dm);
        lw.n2 = up32(find_tensor(tensors, n, pfx + "norm2.weight.tensor").data, dm);
        layers.push_back(lw);
    }
    {
        const auto& tw = find_tensor(tensors, n, "upsample.linear.weight.tensor");
        wu = up16(fold_norm ? fold(tw.data, (size_t)d.upsample_scale * dm, prev_gain)
                            : std::vector<float>(tw.data, tw.data + (size_t)d.upsample_scale * dm * dm));
        bu = up32(find_tensor(tensors, n, "upsample.linear.bias.tensor").data, (size_t)d.upsample_scale * dm);
        const auto& tc_ = find_tensor(tensors, n, "crf.linear.weight.tensor");
        std::vector<float> w((size_t)d.outsize * dm);
        for (size_t i = 0; i < w.size(); ++i) w[i] = tc_.data[i] * d.tx_crf_scale;  // TxModules.cpp:1011-1014
        wc = up16(w);
    }
    {
        // RotaryEmbeddingImpl (TxModules.cpp:184-218): inv_freq via pow in double, angles/cos/sin in fp32
        const int half = 32, tmax = d.max_seq_len > 0 ? d.max_seq_len : 2048;
        std::vector<float> tab((size_t)tmax * half * 2);
        for (int i = 0; i < half; ++i) {
            const float fi = (float)(2 * i) / 64.0f;
            const float inv = (float)(1.0 / std::pow((double)d.theta, (double)fi));
            for (int t = 0; t < tmax; ++t) {
                const float ang = (float)t * inv;
                // position-minor layout [pair of dims j = i / 2][t][(cos, sin) of dim 2j, (cos, sin) of dim 2j + 1]: the GEMM
                // epilogue's 32 lanes hold 32 consecutive positions, so their 16-byte reads of one j are contiguous
                const size_t at = (((size_t)(i >> 1) * tmax + t) * 2 + (i & 1)) * 2;
                tab[at] = std::cos(ang);
                tab[at + 1] = std::sin(ang);
            }
        }
        rope = up32(tab.data(), tab.size());
    }
}

TxModel::~TxModel() {
    for (void* p : owned) cudaFree(p);
}

size_t TxModel::workspace_bytes(int N, int T_in) const {
    const Shapes s = shapes(T_in);
    size_t total = 0;
    auto al = [](size_t b) { return (b + 255) & ~size_t(255); };
    for (int i = 0; i + 1 < desc.num_convs; ++i) total += al((size_t)N * s.t_pad[i] * desc.convs[i].size * 2);
    const size_t rows = (size_t)N * s.t.back();
    total += al(rows * 512 * 2) * 3;                               // x, y, attn out
    total += al(rows * 1536 * 2);                                  // qkv
    total += al(rows * (size_t)desc.dim_feedforward * 2);          // ff hidden
    total += al(rows * (size_t)desc.upsample_scale * 512 * 2);     // upsampled
    total += al(rows * (size_t)gemm_out_ss_parts(512) * 4) * 2;      // partial sums of squares (folded RMSNorm), two in flight
    return total + 4096;
}

std::unique_ptr<ForwardPlan> TxModel::make_plan(int N, int T_in, const __half* signal, __half* scores, void* ws,
                                                size_t ws_bytes) {
    const Shapes s = shapes(T_in);
    const int T = s.t.back();
    if (T > (desc.max_seq_len > 0 ? desc.max_seq_len : 2048)) {
        throw std::invalid_argument("RotE - maximum sequence length exceeded - your chunksize may be too large");
    }
    auto plan = std::make_unique<TxPlan>();
    uint8_t* base = static_cast<uint8_t*>(ws);
    auto take = [&](size_t bytes) {
        uint8_t* p = base;
        base += (bytes + 255) & ~size_t(255);
        if ((size_t)(base - static_cast<uint8_t*>(ws)) > ws_bytes) throw std::logic_error("tx workspace overflow");
        return reinterpret_cast<__half*>(p);
    };
    std::vector<__half*> cbuf;
    for (int i = 0; i + 1 < desc.num_convs; ++i) cbuf.push_back(take((size_t)N * s.t_pad[i] * desc.convs[i].size * 2));
    const long long rows = (long long)N * T;
    __half* x = take((size_t)rows * 512 * 2);
    __half* y = take((size_t)rows * 512 * 2);
    __half* att = take((size_t)rows * 512 * 2);
    __half* qkv = take((size_t)rows * 1536 * 2);
    __half* hid = take((size_t)rows * desc.dim_feedforward * 2);
    __half* ups = take((size_t)rows * desc.upsample_scale * 512 * 2);
    const int ssp = gemm_out_ss_parts(512);
    float* ss_a = reinterpret_cast<float*>(take((size_t)rows * ssp * 4));   // of the rows in x (after fc2 / the previous layer)
    float* ss_b = reinterpret_cast<float*>(take((size_t)rows * ssp * 4));   // of the rows in y (after out_proj)

    plan->conv1 = Conv1Params{signal, cbuf[0], conv1_w, N, T_in, s.t_pad[0], s.pad[0], desc.convs[0].size, desc.convs[0].winlen,
                              desc.convs[0].activation};
    for (int i = 1; i < desc.num_convs; ++i) {
        const auto& c = desc.convs[i];
        GemmDesc g{};
        g.a = cbuf[i - 1];  // row r <-> time r - pad; output t starts at row stride * t
        g.batches = N;
        g.rows_per_batch = s.t[i];
        g.a_row_stride = (int64_t)c.stride * c.insize;
        g.a_batch_stride = (int64_t)s.t_pad[i - 1] * c.insize;
        g.w = conv_w[i - 1];
        g.N = c.size;
        g.K = c.winlen * c.insize;
        g.bias = conv_b[i - 1];
        g.act = c.activation;
        const bool last = i + 1 == desc.num_convs;
        g.out = last ? x : cbuf[i] + (size_t)s.pad[i] * c.size;
        g.out_m1 = s.t[i];
        g.out_s0 = last ? (int64_t)s.t[i] * c.size : (int64_t)s.t_pad[i] * c.size;
        g.out_s1 = c.size;
        plan->convs.push_back(make_gemm_plan(g));
    }
    auto dense = [&](const __half* a, int K, const __half* w, int Nout, const float* bias, int act, __half* out, int ld_out,
                     const __half* residual, float alpha) {
        GemmDesc g{};
        g.a = a;
        g.batches = 1;
        g.rows_per_batch = (int)rows;
        g.a_row_stride = K;
        g.a_batch_stride = (int64_t)rows * K;
        g.w = w;
        g.N = Nout;
        g.K = K;
        g.bias = bias;
        g.act = act;
        g.out = out;
        g.out_m1 = 1;
        g.out_s0 = ld_out;
        g.out_s1 = 0;
        g.residual = residual;
        g.alpha = alpha;
        g.norm_dim = 512;
        if (act == GEMM_ACT_ROPE) {
            g.rope = rope;
            g.rope_T = T;
            g.rope_stride = desc.max_seq_len > 0 ? desc.max_seq_len : 2048;
            g.rope_cols = 2 * desc.nhead * 64;
        }
        return g;
    };
    const int ff = desc.dim_feedforward;
    for (int l = 0; l < desc.depth; ++l) {
        const auto& lw = layers[l];
        TxPlan::Layer L;
        if (fold_norm) {
            // x holds u_prev (un-normalised, ss_a) except before layer 0, y will hold u_mid (ss_b)
            const bool first = l == 0;
            GemmDesc q = dense(x, 512, lw.wqkv, 1536, nullptr, GEMM_ACT_ROPE, qkv, 1536, nullptr, 0.0f);
            if (!first) { q.a_ss = ss_a; q.a_ss_parts = ssp; }
            L.qkv = make_gemm_plan(q);
            GemmDesc o = dense(att, 512, lw.wo, 512, lw.bo, GEMM_ACT_NONE, y, 512, x, desc.deepnorm_alpha);
            if (!first) { o.res_ss = ss_a; o.res_ss_parts = ssp; o.res_gain = layers[l - 1].n2; }
            o.out_ss = ss_b;
            L.out_proj = make_gemm_plan(o);
            GemmDesc f1 = dense(y, 512, lw.w1, 2 * ff, nullptr, GEMM_ACT_SWIGLU, hid, ff, nullptr, 0.0f);
            f1.a_ss = ss_b; f1.a_ss_parts = ssp;
            L.fc1 = make_gemm_plan(f1);
            GemmDesc f2 = dense(hid, ff, lw.w2, 512, nullptr, GEMM_ACT_NONE, x, 512, y, desc.deepnorm_alpha);
            f2.res_ss = ss_b; f2.res_ss_parts = ssp; f2.res_gain = lw.n1;
            f2.out_ss = ss_a;
            L.fc2 = make_gemm_plan(f2);
        } else {
            L.qkv = make_gemm_plan(dense(x, 512, lw.wqkv, 1536, nullptr, GEMM_ACT_ROPE, qkv, 1536, nullptr, 0.0f));
            L.out_proj = make_gemm_plan(dense(att, 512, lw.wo, 512, lw.bo, GEMM_ACT_NONE, y, 512, x, desc.deepnorm_alpha));
            L.fc1 = make_gemm_plan(dense(x, 512, lw.w1, 2 * ff, nullptr, GEMM_ACT_SWIGLU, hid, ff, nullptr, 0.0f));
            L.fc2 = make_gemm_plan(dense(hid, ff, lw.w2, 512, nullptr, GEMM_ACT_NONE, y, 512, x, desc.deepnorm_alpha));
        }
        L.n1 = lw.n1;
        L.n2 = lw.n2;
        plan->layers.push_back(L);
    }
    {
        GemmDesc u = dense(x, 512, wu, desc.upsample_scale * 512, bu, GEMM_ACT_NONE, ups, desc.upsample_scale * 512, nullptr, 0.0f);
        if (fold_norm && desc.depth > 0) { u.a_ss = ss_a; u.a_ss_parts = ssp; }
        plan->upsample = make_gemm_plan(u);
    }
    {
        GemmDesc g{};
        g.a = ups;
        g.batches = 1;
        g.rows_per_batch = (int)(rows * desc.upsample_scale);
        g.a_row_stride = 512;
        g.a_batch_stride = (int64_t)rows * desc.upsample_scale * 512;
        g.w = wc;
        g.N = desc.outsize;
        g.K = 512;
        g.act = GEMM_ACT_NONE;
        g.out = scores;
        g.out_m1 = 1;
        g.out_s0 = desc.outsize;
        plan->crf = make_gemm_plan(g);
    }
    plan->qkv_map = make_tmap_2d(qkv, (uint64_t)3 * desc.nhead * ATT_D, (uint64_t)rows, (uint64_t)3 * desc.nhead * ATT_D * 2, ATT_D, 128);
    if (desc.attn_window_upper > AT_BK || desc.attn_window_lower > AT_BK || desc.attn_window_upper < 0 || desc.attn_window_lower < 0) {
        throw Unsupported("attention window must lie within [-128, +128] (three key blocks per query tile)");
    }
    plan->attn_tc_p = AttnTcParams{att, N, T, desc.nhead, desc.attn_window_upper, desc.attn_window_lower};
    plan->x = x;
    plan->y = y;
    plan->rows = rows;
    plan->N = N;
    plan->T = T;
    plan->H = desc.nhead;
    plan->fold_norm = fold_norm;
    plan->n_launches = 1 + (desc.num_convs - 1) + desc.depth * (fold_norm ? 5 : 7) + 2;
    return plan;
}

void TxPlan::run(cudaStream_t stream, ProfileSink* prof) {
    nvtxRangePushA("Conv");
    {
        const long long total = (long long)conv1.N * conv1.T * (conv1.C1 / 8);
        tx_conv1_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(conv1);
        if (prof) prof->mark("tx_conv1", stream);
    }
    for (auto& c : convs) {
        run_gemm(c, stream);
        if (prof) prof->mark("tx_conv_gemm", stream);
    }
    nvtxRangePop();
    const unsigned norm_grid = (unsigned)((rows + 7) / 8);
    nvtxRangePushA("TransEnc");
    for (auto& L : layers) {
        NvtxRange layer("TxLayerKoiTiled");
        {
            NvtxRange r("QKV+ROTE");
            run_gemm(L.qkv, stream);
            if (prof) prof->mark("qkv_gemm", stream);
        }
        {
            NvtxRange r("MEA");
            constexpr int smem = AT_SMEM;
            ensure_dynamic_smem(tx_attention_tc_kernel, smem);
            tx_attention_tc_kernel<<<dim3((unsigned)((T + AT_BQ - 1) / AT_BQ), (unsigned)H, (unsigned)N), AT_THREADS, smem, stream>>>(qkv_map, attn_tc_p);
            if (prof) prof->mark("tx_attention", stream);
        }
        {
            NvtxRange r("OUTP");
            run_gemm(L.out_proj, stream);
            if (prof) prof->mark("out_proj_gemm", stream);
        }
        if (!fold_norm) {
            NvtxRange r("LNORM1");
            rmsnorm512_kernel<<<norm_grid, 256, 0, stream>>>(y, x, L.n1, rows);
            if (prof) prof->mark("rmsnorm", stream);
        }
        {
            NvtxRange r("FC1+SILU");
            run_gemm(L.fc1, stream);
            if (prof) prof->mark("fc1_swiglu_gemm", stream);
        }
        {
            NvtxRange r("FC2");
            run_gemm(L.fc2, stream);
            if (prof) prof->mark("fc2_gemm", stream);
        }
        if (!fold_norm) {
            NvtxRange r("LNORM2");
            rmsnorm512_kernel<<<norm_grid, 256, 0, stream>>>(y, x, L.n2, rows);
            if (prof) prof->mark("rmsnorm", stream);
        }
    }
    nvtxRangePop();
    {
        NvtxRange r("TransDec");
        run_gemm(upsample, stream);
        if (prof) prof->mark("upsample_gemm", stream);
    }
    {
        NvtxRange r("CRF");
        run_gemm(crf, stream);
        if (prof) prof->mark("crf_gemm", stream);
    }
    B200_CUDA(cudaGetLastError());
}

}  // namespace

std::unique_ptr<Model> make_tx_model(const b200_model_desc& desc, const b200_tensor* tensors, int n) {
    return std::make_unique<TxModel>(desc, tensors, n);
}

}  // namespace b200
