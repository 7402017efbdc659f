// Conv -> Transformer encoder -> upsample -> scaled CRF linear forward (sup models, and d_model up to 1536 with
// windows up to +-256, e.g. the 1536-wide / 24-head / (255, 256) encoder) for sm_90a.
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
//
// Precision B200_TX_FP8_FFN (the reference's koi_use_f8 = 1, koi_use_i8 = 0 configuration, TxModules.cpp:477-479, 560-575,
// 596-697): fc1 and fc2 take E4M3 operands.  norm1 is an explicit pass that writes the fp16 row (fc2's residual) and its
// E4M3 copy (fc1's A); fc1 + SwiGLU writes E4M3 (fc2's A); fc2 writes fp16.  The fp16 weights the reference keeps (QKV,
// out_proj, both RMSNorm gains) lose their low 4 mantissa bits first (remove_bits, TxModules.cpp:104-111, 443-453).
//
// Precision B200_TX_I8_QKV_FP8_FFN (koi_use_f8 = 1 with koi_use_i8 = 1, the reference's default on an H100: TxModules.cpp:477-479,
// 936-961, 497-506, 611-616, 669, 713): as fp8_ffn, but the fused QKV + RoPE projection takes int8 operands.  Wqkv is
// quantised per output row from the fp16 weights before remove_bits; the stack's input is quantised per token row by a device
// pass, and norm2 becomes an explicit pass that writes the next layer's fp16 rows and their int8 copy.  Nothing is folded:
// out_proj's residual and the upsample read the normalised fp16 rows.
#include "engine.h"
#include "gemm.h"
#include "nvtx.h"

#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>

namespace b200 {

std::vector<float> rope_table(float theta, int tmax) {
    // RotaryEmbeddingImpl (TxModules.cpp:184-218): inv_freq via pow in double, angles/cos/sin in fp32
    const int half = 32;
    std::vector<float> tab((size_t)tmax * half * 2);
    for (int i = 0; i < half; ++i) {
        const float fi = (float)(2 * i) / 64.0f;
        const float inv = (float)(1.0 / std::pow((double)theta, (double)fi));
        for (int t = 0; t < tmax; ++t) {
            const float ang = (float)t * inv;
            // position-minor layout [pair of dims j = i / 2][t][(cos, sin) of dim 2j, (cos, sin) of dim 2j + 1]: the GEMM
            // epilogue's 32 lanes hold 32 consecutive positions, so their 16-byte reads of one j are contiguous
            const size_t at = (((size_t)(i >> 1) * tmax + t) * 2 + (i & 1)) * 2;
            tab[at] = std::cos(ang);
            tab[at + 1] = std::sin(ang);
        }
    }
    return tab;
}

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
// Per-row int8 quantisation of fp16 rows (the QKV projection's A in the int8_qkv_fp8_ffn precision), by the warp of a row
// whose lane holds `per` consecutive columns from src (absmax: the largest |x| of the lane's columns): utils::quantize_tensor
// (tensor_utils.cpp:293-300) as torch evaluates it on fp16, i.e. quantize_rows_f16's arithmetic --
//     scale16 = fp16(128 / absmax)   q = clip(rne(fp16(x * scale16)), -127, 127)   inv = 1 / float(scale16)
// with the reference's reciprocal of the scale (TxModules.cpp:958).  An all-zero row gets q = 0; a row whose scale overflows
// to +inf (absmax 0, or below about 128 / 65520) gets inv = 0, and there a zero element's product 0 * inf is NaN, which the
// clip takes to -127 as quantize_rows_f16 does (fmaxf, std::max): q is defined everywhere and such rows contribute 0.
__device__ __forceinline__ void quantize_row_i8(const __half* src, int per, float absmax, int lane, int8_t* q, float* inv) {
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) absmax = fmaxf(absmax, __shfl_xor_sync(0xffffffffu, absmax, o));
    const float scale = __half2float(__float2half_rn(__fdiv_rn(128.0f, absmax)));
    if (lane == 0) *inv = __fdiv_rn(1.0f, scale);
    for (int i = 0; i < per; i += 4) {
        const uint2 v = *reinterpret_cast<const uint2*>(src + i);
        const __half* h = reinterpret_cast<const __half*>(&v);
        uint32_t packed = 0;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            int qv = 0;
            if (absmax != 0.0f) {
                const float prod = __half2float(__float2half_rn(__fmul_rn(__half2float(h[e]), scale)));
                qv = (int)fminf(127.0f, fmaxf(-127.0f, rintf(prod)));
            }
            packed |= (uint32_t)(qv & 0xff) << (8 * e);
        }
        *reinterpret_cast<uint32_t*>(q + i) = packed;
    }
}

// The stack input's int8 copy (int8_qkv_fp8_ffn): quantize_row_i8 of every fp16 row of in [rows][dim], one warp per row
__global__ void __launch_bounds__(256) quantize_i8_kernel(const __half* __restrict__ in, long long rows, int dim,
                                                          int8_t* __restrict__ q, float* __restrict__ inv) {
    const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const int per = dim / 32;
    const __half* src = in + row * dim + lane * per;
    float absmax = 0.0f;
    for (int i = 0; i < per; i += 4) {
        const uint2 v = *reinterpret_cast<const uint2*>(src + i);
        const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const float2 a = __half22float2(h[j]);
            absmax = fmaxf(absmax, fmaxf(fabsf(a.x), fabsf(a.y)));
        }
    }
    quantize_row_i8(src, per, absmax, lane, q + row * dim + lane * per, inv + row);
}

// ------------------------------------------------------------------------------------------------
// RMSNorm over rows of `dim` (RMSNorm.cpp:14-18): x * rsqrt(mean(x^2) + eps) * w ; one warp per row, lane i owns the dim / 32
// consecutive columns from i * dim / 32 (dim a multiple of 128, so whole 8-byte groups).  The row is read twice (sum of
// squares, then the scaled store) rather than held in registers, so one kernel serves every width.
// ------------------------------------------------------------------------------------------------
// out8 (optional): the E4M3 cast of the fp16 values written to out, same layout (fc1's A in the fp8_ffn precision).
// outq / out_inv (optional): quantize_row_i8 of the fp16 values written to out (norm2 in the int8_qkv_fp8_ffn precision: the
// next QKV projection's A).  Koi's requantisation inside koi_rmsnorm_residual is closed source; quantising the stored fp16
// row with the stack input's arithmetic is this engine's choice.
__global__ void __launch_bounds__(256) rmsnorm_kernel(const __half* __restrict__ in, __half* __restrict__ out,
                                                      const float* __restrict__ w, long long rows, int dim,
                                                      uint8_t* __restrict__ out8, int8_t* __restrict__ outq,
                                                      float* __restrict__ out_inv) {
    const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const int per = dim / 32;
    const __half* src = in + row * dim + lane * per;
    float ss = 0.0f;
    for (int i = 0; i < per; i += 4) {
        const uint2 v = *reinterpret_cast<const uint2*>(src + i);
        const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const float2 a = __half22float2(h[j]);
            ss += a.x * a.x + a.y * a.y;
        }
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float rstd = rsqrtf(ss * (1.0f / (float)dim) + 1e-5f);
    __half* dst = out + row * dim + lane * per;
    float absmax = 0.0f;   // of the fp16 values stored (outq)
    for (int i = 0; i < per; i += 4) {
        const uint2 v = *reinterpret_cast<const uint2*>(src + i);
        const __half2* h = reinterpret_cast<const __half2*>(&v);
        __half2 o2[2];
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int c = lane * per + i + 2 * j;
            const float2 a = __half22float2(h[j]);
            o2[j] = __floats2half2_rn(a.x * rstd * __ldg(w + c), a.y * rstd * __ldg(w + c + 1));
        }
        *reinterpret_cast<uint2*>(dst + i) = *reinterpret_cast<uint2*>(o2);
        if (outq) {
            const float2 f0 = __half22float2(o2[0]), f1 = __half22float2(o2[1]);
            absmax = fmaxf(absmax, fmaxf(fmaxf(fabsf(f0.x), fabsf(f0.y)), fmaxf(fabsf(f1.x), fabsf(f1.y))));
        }
        if (out8) {
            const float2 f0 = __half22float2(o2[0]), f1 = __half22float2(o2[1]);
            const uint32_t q = (uint32_t)tc::cvt_e4m3x2(f0.x, f0.y) | ((uint32_t)tc::cvt_e4m3x2(f1.x, f1.y) << 16);
            *reinterpret_cast<uint32_t*>(out8 + row * dim + lane * per + i) = q;
        }
    }
    // the lane reads back its own stores
    if (outq) quantize_row_i8(dst, per, absmax, lane, outq + row * dim + lane * per, out_inv + row);
}

constexpr int ATT_D = 64;   // head dimension

// ------------------------------------------------------------------------------------------------
// Sliding-window attention on the tensor cores (successor of koi_masked_attention, TxModules.cpp:648; window semantics
// TxModules.cpp:310-317: keys j with -win_upper <= j - i <= win_lower).
// qkv: [N*T][3][H][64] fp16 (output of the Wqkv GEMM, q and k already rotated); out: [N*T][H*64] fp16.
// One CTA = 128 queries of one (chunk, head); the keys they can see lie in at most AT_MAXBLK aligned blocks of 128 keys
// (5 for windows up to 256 on either side: 3 for sup's (127, 128)).  Thread 0 loads Q and the K / V blocks by TMA (128-byte
// swizzle) into a ring of AT_SLOTS slots; each of the eight warps owns 16 query rows and walks the blocks flash-style on
// mma.sync:
//     S_b = Q K_b^T          16 x 128 per warp, fp32 in registers (Q and K_b fragments by ldmatrix)
//     P_b = exp2(S_b' - m)   running max / sum per row (the four lanes of a quad share a row), P rounded to fp16 and
//                            re-used in registers as the A fragments of the next product
//     O = O * alpha + P_b V_b  V_b as it lies in memory ([key][d]) through ldmatrix.trans -- no transposed copy of V
// Blocks beyond the third stream through the ring: every warp arrives on its slot's "empty" barrier when it is done with
// a block, and thread 0 then refills the slot with the block AT_SLOTS further on.  A warp none of whose rows sees a block
// skips its arithmetic (masked out, the block would leave o, l_run and -- after a visible block -- m_run unchanged).
// Shared memory 113 KB (Q and three K / V slots) for every window, and at most 128 registers (__launch_bounds__ min 2).
// ------------------------------------------------------------------------------------------------
constexpr int AT_BQ = 128, AT_BK = 128;
constexpr int AT_TILE = 128 * 64 * 2;   // one [128 x 64] fp16 tile
constexpr int AT_MAX_WIN = 256;         // largest win_upper / win_lower the host accepts
constexpr int AT_MAXBLK = 1 + (AT_MAX_WIN + AT_BK - 1) / AT_BK + (AT_BQ - 1 + AT_MAX_WIN) / AT_BK;   // 5
constexpr int AT_SLOTS = 3;             // K / V ring slots
constexpr int AT_THREADS = 256;
constexpr int AT_SMEM = 1024 + (1 + 2 * AT_SLOTS) * AT_TILE + 64;
static_assert((1 + 2 * AT_SLOTS) * 8 <= 64, "mbarriers do not fit their 64 bytes");
static_assert(AT_MAXBLK == 5, "a 128-query tile of a +-256 window spans five key blocks");

struct AttnTcParams {
    __half* out;   // [N*T][H*64]
    int N, T, H;
    int win_upper, win_lower;
};

__global__ void __launch_bounds__(AT_THREADS, 2) tx_attention_tc_kernel(const __grid_constant__ CUtensorMap tma_qkv, const AttnTcParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* q_s = smem;                          // [128 q][64 d]
    uint8_t* k_s = q_s + AT_TILE;                 // [AT_SLOTS][128 keys][64 d]
    uint8_t* v_s = k_s + AT_SLOTS * AT_TILE;      // [AT_SLOTS][128 keys][64 d]
    uint64_t* bars = reinterpret_cast<uint64_t*>(v_s + AT_SLOTS * AT_TILE);
    uint64_t* q_full = bars;                      // TMA -> warps
    uint64_t* kv_full = bars + 1;                 // [AT_SLOTS] TMA -> warps
    uint64_t* kv_empty = kv_full + AT_SLOTS;      // [AT_SLOTS] warps -> thread 0 (one arrival per warp)

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int qt = blockIdx.x, h = blockIdx.y, n = blockIdx.z;
    const int q0 = qt * AT_BQ;
    // aligned key blocks that intersect [q0 - win_upper, q0 + 127 + win_lower] and [0, T)
    int kb_first = (q0 - p.win_upper) / AT_BK;   // q0 >= 0, so this only goes negative through the subtraction
    if (q0 - p.win_upper < 0) kb_first = 0;
    int kb_last = (q0 + AT_BQ - 1 + p.win_lower) / AT_BK;
    const int kb_max = (p.T - 1) / AT_BK;
    if (kb_last > kb_max) kb_last = kb_max;
    const int nblk = kb_last - kb_first + 1;     // 1..AT_MAXBLK (windows checked on the host)
    const int row0 = n * p.T;   // first token row of this chunk in the [N*T][3 * H * 64] view
    // K and V of block b into ring slot b % AT_SLOTS
    auto load_kv = [&](int b) {
        const int s = b % AT_SLOTS;
        tc::mbar_arrive_expect_tx(&kv_full[s], 2 * AT_TILE);
        const int krow = row0 + (kb_first + b) * AT_BK;
        tc::tma_load_2d(k_s + s * AT_TILE, &tma_qkv, &kv_full[s], (p.H + h) * ATT_D, krow);
        tc::tma_load_2d(v_s + s * AT_TILE, &tma_qkv, &kv_full[s], (2 * p.H + h) * ATT_D, krow);
    };

    if (threadIdx.x == 0) {
        tc::mbar_init(q_full, 1);
        for (int i = 0; i < AT_SLOTS; ++i) {
            tc::mbar_init(&kv_full[i], 1);
            tc::mbar_init(&kv_empty[i], AT_THREADS / 32);
        }
        tc::fence_barrier_init();
        tc::prefetch_tmap(&tma_qkv);
        tc::mbar_arrive_expect_tx(q_full, AT_TILE);
        tc::tma_load_2d(q_s, &tma_qkv, q_full, h * ATT_D, row0 + q0);
        for (int b = 0; b < nblk && b < AT_SLOTS; ++b) load_kv(b);
    }
    __syncthreads();

    const int qm = lane >> 3, qr = lane & 7;   // ldmatrix.x4: matrix qm, row qr
    const int quad = lane & 3;
    const float sc = 0.125f * 1.44269504088896341f;   // 1/sqrt(64) and the base change of exp -> exp2
    int qi[2];
    qi[0] = q0 + warp * 16 + (lane >> 2);
    qi[1] = qi[0] + 8;
    tc::mbar_wait_silent(q_full, 0);
    float o[ATT_D / 8][4];
#pragma unroll
    for (int dt = 0; dt < ATT_D / 8; ++dt) o[dt][0] = o[dt][1] = o[dt][2] = o[dt][3] = 0.0f;
    float m_run[2] = {-1e30f, -1e30f}, l_run[2] = {0.0f, 0.0f};

    for (int b = 0; b < nblk; ++b) {
        const int slot = b % AT_SLOTS;
        const uint32_t ring_phase = (uint32_t)(b / AT_SLOTS) & 1u;
        const int kb = (kb_first + b) * AT_BK;
        const uint8_t* kt = k_s + slot * AT_TILE;
        const uint8_t* vt = v_s + slot * AT_TILE;
        // keys of this block visible to each row: j in [lo, hi)
        int lo[2], hi[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            lo[r] = max(qi[r] - p.win_upper - kb, 0);
            hi[r] = min(min(qi[r] + p.win_lower + 1 - kb, AT_BK), p.T - kb);
            if (qi[r] >= p.T) hi[r] = 0;
        }
        // every warp waits for the block, so that no load is still in flight when thread 0 re-arms the slot
        tc::mbar_wait_silent(&kv_full[slot], ring_phase);
        if (__any_sync(0xffffffffu, hi[0] > lo[0] || hi[1] > lo[1])) {
            // S = Q K^T: 16 key tiles of 8; K fragments: matrix qm = (key tile 2 np + qm / 2, d half qm % 2)
            float sacc[AT_BK / 8][4];
#pragma unroll
            for (int nt = 0; nt < AT_BK / 8; ++nt) sacc[nt][0] = sacc[nt][1] = sacc[nt][2] = sacc[nt][3] = 0.0f;
#pragma unroll
            for (int ks = 0; ks < ATT_D / 16; ++ks) {
                // A fragment of this warp's 16 query rows, d 16 ks .. + 15 (re-read from the resident Q tile: keeping all
                // four in registers across the block loop doubles the spills); matrix qm = (row half qm % 2, d half qm / 2)
                uint32_t qa[4];
                tc::ldmatrix_x4(qa, tc::smem_u32(q_s + tc::sw128_offset(warp * 16 + (qm & 1) * 8 + qr, 2 * ks + (qm >> 1))));
#pragma unroll
                for (int np = 0; np < AT_BK / 16; ++np) {
                    uint32_t kf[4];
                    tc::ldmatrix_x4(kf, tc::smem_u32(kt + tc::sw128_offset((2 * np + (qm >> 1)) * 8 + qr, 2 * ks + (qm & 1))));
                    tc::mma_f16_16816(sacc[2 * np], qa, kf[0], kf[1]);
                    tc::mma_f16_16816(sacc[2 * np + 1], qa, kf[2], kf[3]);
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
        }   // any row of the warp sees the block
        // release the slot; once all eight warps have, thread 0 refills it with block b + AT_SLOTS
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&kv_empty[slot]);
        if (threadIdx.x == 0 && b + AT_SLOTS < nblk) {
            tc::mbar_wait_silent(&kv_empty[slot], ring_phase);
            load_kv(b + AT_SLOTS);
        }
        __syncwarp();
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

// Windows the kernel handles: every key band of a query tile spans at most AT_MAXBLK blocks.
void check_attention_window(int win_upper, int win_lower) {
    if (win_upper < 0 || win_lower < 0 || win_upper > AT_MAX_WIN || win_lower > AT_MAX_WIN) {
        throw Unsupported("attention window must lie within [-256, +256] (at most five key blocks per query tile), got (" +
                          std::to_string(win_upper) + ", " + std::to_string(win_lower) + ")");
    }
}

// The attention launch of the model and of the kernel-level test hook.
void launch_attention(const CUtensorMap& qkv_map, const AttnTcParams& p, cudaStream_t stream) {
    ensure_dynamic_smem(tx_attention_tc_kernel, AT_SMEM);
    tx_attention_tc_kernel<<<dim3((unsigned)((p.T + AT_BQ - 1) / AT_BQ), (unsigned)p.H, (unsigned)p.N), AT_THREADS, AT_SMEM, stream>>>(
            qkv_map, p);
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
struct TxLayerWeights {
    __half *wqkv = nullptr, *wo = nullptr, *w1 = nullptr, *w2 = nullptr;
    uint8_t *w1_e4m3 = nullptr, *w2_e4m3 = nullptr;   // fp8_ffn: fc1 (interleaved rows) and fc2 as E4M3 (w1, w2 unused)
    int8_t* wqkv_i8 = nullptr;                         // int8_qkv_fp8_ffn: Wqkv per output row (wqkv unused)
    float* wqkv_inv = nullptr;                         // and the fp32 factor 1 / float(scale16) of each row
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
    std::string info() const override { return i8 ? "tx.fp8_ffn=1;tx.int8_qkv=1" : fp8 ? "tx.fp8_ffn=1" : std::string(); }
    std::vector<Layer> layers;
    GemmPlan upsample, crf;
    CUtensorMap qkv_map;       // qkv as [N*T][3*H*64], box 64 x 128 (Q, K and V tiles of the tensor-core attention)
    AttnTcParams attn_tc_p{};
    __half *x = nullptr, *y = nullptr;
    long long rows = 0;
    int N = 0, T = 0, H = 0;
    int norm_dim = 0;   // d_model: row width of the separate RMSNorm pass
    int n_launches = 0;
    int stop_after = -1;        // B200_DEBUG_TX_LAUNCHES: run() returns after this many launches (-1: the whole plan)
    bool fold_norm = true;
    bool fp8 = false;           // fp8_ffn: explicit norm1 pass writing fp16 (norm_out) and E4M3 (norm_out8), E4M3 fc1 / fc2
    bool i8 = false;            // int8_qkv_fp8_ffn (fp8 set too): stack input quantise pass, norm2 writing x8 / x_inv, int8 qkv
    __half* norm_out = nullptr;
    uint8_t* norm_out8 = nullptr;
    int8_t* x8 = nullptr;       // int8 copy of x's rows and their factors (int8_qkv_fp8_ffn)
    float* x_inv = nullptr;
};

class TxModel final : public Model {
public:
    TxModel(const b200_model_desc& d, const b200_tensor* tensors, int n);
    ~TxModel() override;
    size_t workspace_bytes(int N, int T_in) const override;
    std::unique_ptr<ForwardPlan> make_plan(int N, int T_in, const __half* signal, __half* scores, void* ws,
                                           size_t ws_bytes) override;
    b200_model_desc desc;
    // B200_TX_RMSNORM_PASS=1: separate RMSNorm kernel after every sub-layer (A/B comparisons).  false in int8_qkv_fp8_ffn,
    // where both norms are explicit passes and no gain is folded into a weight
    bool fold_norm = true;
    bool fp8 = false;        // B200_TX_FP8_FFN or B200_TX_I8_QKV_FP8_FFN (fp8_ffn: norm2 stays folded; the RMSNorm-pass option is ignored)
    bool i8 = false;         // B200_TX_I8_QKV_FP8_FFN
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
    struct Buffers {
        std::vector<__half*> cbuf;  // output of conv i (but the last), [N][t_pad[i]][size]
        __half *x, *y, *att, *qkv, *hid, *ups;
        float *ss_a, *ss_b;  // partial sums of squares (folded RMSNorm) of the rows in x and in y
        int8_t* x8;          // int8_qkv_fp8_ffn: the int8 copy of x's rows [rows][d_model] and their factors [rows]
        float* x_inv;        // (both null in the other precisions)
    };
    // The workspace layout for N chunks of T_in samples; refuses a chunk longer than the RoPE table
    Buffers carve(Bump& b, int N, int T_in) const;
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
    i8 = d.tx_precision == B200_TX_I8_QKV_FP8_FFN;
    fp8 = d.tx_precision == B200_TX_FP8_FFN || i8;
    if (const char* e = std::getenv("B200_TX_RMSNORM_PASS"); e && !fp8) fold_norm = std::atoi(e) == 0;
    if (i8) fold_norm = false;
    // the shapes the kernels handle: head dimension 64 (attention, RoPE epilogue), d_model in whole 128-column tiles (the
    // folded RMSNorm's partial sums), K of the fc2 GEMM in whole 64-wide blocks, key bands of at most AT_MAXBLK blocks
    if (d.nhead < 1 || d.d_model != ATT_D * d.nhead) throw Unsupported("transformer path needs d_model == 64 * nhead (head dimension 64)");
    if (d.d_model % 128 != 0 || d.d_model > 1536) throw Unsupported("transformer path needs d_model a multiple of 128 and at most 1536");
    if (d.dim_feedforward < 64 || d.dim_feedforward % 64 != 0) throw Unsupported("transformer path needs dim_feedforward a multiple of 64");
    check_attention_window(d.attn_window_upper, d.attn_window_lower);
    if (fp8 && d.dim_feedforward % 128 != 0) {
        throw Unsupported(std::string(i8 ? "int8_qkv_fp8_ffn" : "fp8_ffn") +
                          " precision needs dim_feedforward a multiple of 128 (fc2's K in whole 128-byte E4M3 blocks)");
    }
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
    // fp8_ffn: the model as the reference holds it, fp16 (CudaCaller.cpp:167), with remove_bits applied to the fp16 weights
    // it keeps; E4M3 weights are cast from the fp16 values.  The gains are rounded before they are folded into columns.
    std::vector<std::vector<float>> rounded;   // this layer's weights as the engine uses them (rounded in fp8_ffn)
    std::vector<float> gain2;                  // storage of prev_gain
    auto rb = [&](const float* v, size_t cnt) -> const float* {
        rounded.push_back(fp8 ? fp16_remove_bits(v, cnt, 4) : std::vector<float>(v, v + cnt));
        return rounded.back().data();
    };
    auto up_bytes = [&](const void* data, size_t cnt) {
        void* p = nullptr;
        B200_CUDA(cudaMalloc(&p, cnt));
        owned.push_back(p);
        B200_CUDA(cudaMemcpy(p, data, cnt, cudaMemcpyHostToDevice));
        return p;
    };
    auto up8 = [&](const float* v, size_t cnt) {
        std::vector<uint8_t> q(cnt);
        for (size_t i = 0; i < cnt; ++i) q[i] = e4m3_from_f16_bits(f16_bits(v[i]));
        return static_cast<uint8_t*>(up_bytes(q.data(), cnt));
    };
    for (int l = 0; l < d.depth; ++l) {
        const std::string pfx = "transformer_encoder." + std::to_string(l) + ".";
        TxLayerWeights lw;
        const float* n1 = rb(find_tensor(tensors, n, pfx + "norm1.weight.tensor").data, dm);
        const float* n2 = rb(find_tensor(tensors, n, pfx + "norm2.weight.tensor").data, dm);
        const auto& wqkv_t = find_tensor(tensors, n, pfx + "self_attn.Wqkv.weight.tensor");
        if (i8) {
            // quantize_tensor(fp16(Wqkv), -1), one scale per output row, from the fp16 weights as they are BEFORE remove_bits
            // (the reference quantises at TxModules.cpp:499 and rounds at :589); its Q / K row interleave (:488-496) moves
            // rows without changing any, so the engine's row order stays.  No gain in the columns: norm2 is a pass here.
            const size_t cnt = (size_t)3 * dm * dm;
            std::vector<uint16_t> h(cnt);
            for (size_t i = 0; i < cnt; ++i) h[i] = f16_bits(wqkv_t.data[i]);
            std::vector<int8_t> q(cnt);
            std::vector<uint16_t> scale((size_t)3 * dm);
            quantize_rows_f16(h.data(), 3 * dm, dm, q.data(), scale.data());
            std::vector<float> inv((size_t)3 * dm);
            for (int r = 0; r < 3 * dm; ++r) {
                __half_raw raw;
                raw.x = scale[r];
                inv[r] = 1.0f / __half2float(__half(raw));   // scale.reciprocal_(): 0 for an infinite scale
            }
            lw.wqkv_i8 = reinterpret_cast<int8_t*>(up_bytes(q.data(), cnt));
            lw.wqkv_inv = up32(inv.data(), inv.size());
        } else {
            const float* wqkv = rb(wqkv_t.data, (size_t)3 * dm * dm);
            lw.wqkv = up16(fold_norm ? fold(wqkv, (size_t)3 * dm, prev_gain) : std::vector<float>(wqkv, wqkv + (size_t)3 * dm * dm));
        }
        const float* wo = rb(find_tensor(tensors, n, pfx + "self_attn.out_proj.weight.tensor").data, (size_t)dm * dm);
        lw.wo = up16(std::vector<float>(wo, wo + (size_t)dm * dm));
        lw.bo = up32(find_tensor(tensors, n, pfx + "self_attn.out_proj.bias.tensor").data, dm);
        // fc1 rows [y(0..ff) | gate(0..ff)] (TxModules.cpp:170-176) interleaved to (y_j, gate_j) pairs
        const auto& w1 = find_tensor(tensors, n, pfx + "ff.fc1.weight.tensor");
        std::vector<float> w1i((size_t)2 * ff * dm);
        for (int j = 0; j < ff; ++j) {
            std::memcpy(&w1i[(size_t)(2 * j) * dm], &w1.data[(size_t)j * dm], sizeof(float) * dm);
            std::memcpy(&w1i[(size_t)(2 * j + 1) * dm], &w1.data[(size_t)(ff + j) * dm], sizeof(float) * dm);
        }
        const auto& w2 = find_tensor(tensors, n, pfx + "ff.fc2.weight.tensor");
        if (fp8) {
            // norm1 is an explicit pass here, so no gain goes into fc1's columns
            lw.w1_e4m3 = up8(w1i.data(), w1i.size());
            lw.w2_e4m3 = up8(w2.data, (size_t)dm * ff);
        } else {
            lw.w1 = up16(fold_norm ? fold(w1i.data(), (size_t)2 * ff, n1) : w1i);
            lw.w2 = up16(std::vector<float>(w2.data, w2.data + (size_t)dm * ff));
        }
        lw.n1 = up32(n1, dm);
        lw.n2 = up32(n2, dm);
        layers.push_back(lw);
        gain2.assign(n2, n2 + dm);
        prev_gain = gain2.data();
        rounded.clear();
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
        const std::vector<float> tab = rope_table(d.theta, d.max_seq_len > 0 ? d.max_seq_len : 2048);
        rope = up32(tab.data(), tab.size());
    }
}

TxModel::~TxModel() {
    for (void* p : owned) cudaFree(p);
}

TxModel::Buffers TxModel::carve(Bump& b, int N, int T_in) const {
    const Shapes s = shapes(T_in);
    const int T = s.t.back();
    if (T > (desc.max_seq_len > 0 ? desc.max_seq_len : 2048)) {
        throw std::invalid_argument("RotE - maximum sequence length exceeded - your chunksize may be too large");
    }
    Buffers w;
    for (int i = 0; i + 1 < desc.num_convs; ++i) w.cbuf.push_back(b.take<__half>((size_t)N * s.t_pad[i] * desc.convs[i].size * 2));
    const size_t rows = (size_t)N * T, dm = desc.d_model;
    w.x = b.take<__half>(rows * dm * 2);
    w.y = b.take<__half>(rows * dm * 2);
    w.att = b.take<__half>(rows * dm * 2);
    w.qkv = b.take<__half>(rows * 3 * dm * 2);
    w.hid = b.take<__half>(rows * desc.dim_feedforward * 2);
    w.ups = b.take<__half>(rows * desc.upsample_scale * dm * 2);
    w.ss_a = b.take<float>(rows * gemm_out_ss_parts((int)dm) * 4);   // x: after fc2 / the previous layer
    w.ss_b = b.take<float>(rows * gemm_out_ss_parts((int)dm) * 4);   // y: after out_proj
    w.x8 = nullptr;
    w.x_inv = nullptr;
    if (i8) {
        // their own blocks: x8 lives from norm2 (or the stack input's quantise pass) to the next QKV projection, which writes
        // qkv and so cannot share it, while the other buffers it could share are not provably as large for every shape
        w.x8 = b.take<int8_t>(rows * dm);
        w.x_inv = b.take<float>(rows * 4);
    }
    return w;
}

size_t TxModel::workspace_bytes(int N, int T_in) const {
    Bump sizing;
    carve(sizing, N, T_in);
    return sizing.used();
}

std::unique_ptr<ForwardPlan> TxModel::make_plan(int N, int T_in, const __half* signal, __half* scores, void* ws,
                                                size_t ws_bytes) {
    const Shapes s = shapes(T_in);
    const int T = s.t.back();
    Bump b(ws, ws_bytes);
    const auto [cbuf, x, y, att, qkv, hid, ups, ss_a, ss_b, x8, x_inv] = carve(b, N, T_in);
    if (b.used() != ws_bytes) throw std::logic_error("tx workspace: the plan's layout differs from workspace_bytes()");
    auto plan = std::make_unique<TxPlan>();
    const long long rows = (long long)N * T;
    const int dm = desc.d_model, dqkv = 3 * desc.d_model;
    const int ssp = gemm_out_ss_parts(dm);

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
    auto dense = [&](const void* a, int K, const void* w, int Nout, const float* bias, int act, void* out, int ld_out,
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
        g.norm_dim = dm;
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
        if (i8) {
            // x holds the normalised rows (the conv output before layer 0) and x8 / x_inv their int8 copy.  qkv: int8 x int8
            // with RoPE; out_proj -> y (+ alpha * x); norm1 y -> att (fp16) + qkv's buffer (E4M3); fc1 + SwiGLU -> hid
            // (E4M3); fc2 -> y (+ alpha * att); norm2 y -> x (fp16) + x8 / x_inv
            GemmDesc q = dense(x8, dm, lw.wqkv_i8, dqkv, nullptr, GEMM_ACT_ROPE, qkv, dqkv, nullptr, 0.0f);
            q.in_type = GEMM_S8;
            q.row_scale = x_inv;
            q.col_scale = lw.wqkv_inv;
            L.qkv = make_gemm_plan(q);
            L.out_proj = make_gemm_plan(dense(att, dm, lw.wo, dm, lw.bo, GEMM_ACT_NONE, y, dm, x, desc.deepnorm_alpha));
            GemmDesc f1 = dense(qkv, dm, lw.w1_e4m3, 2 * ff, nullptr, GEMM_ACT_SWIGLU, hid, ff, nullptr, 0.0f);
            f1.in_type = GEMM_E4M3;
            f1.out_type = GEMM_E4M3;
            L.fc1 = make_gemm_plan(f1);
            GemmDesc f2 = dense(hid, ff, lw.w2_e4m3, dm, nullptr, GEMM_ACT_NONE, y, dm, att, desc.deepnorm_alpha);
            f2.in_type = GEMM_E4M3;
            L.fc2 = make_gemm_plan(f2);
        } else if (fp8) {
            // qkv and out_proj as in the folded fp16 layout; norm1 -> att (fp16) + qkv's buffer (E4M3, free once attention has
            // read it); fc1 + SwiGLU -> hid (E4M3); fc2 -> x (fp16, + alpha * att) with the partial sums for the folded norm2
            const bool first = l == 0;
            GemmDesc q = dense(x, dm, lw.wqkv, dqkv, nullptr, GEMM_ACT_ROPE, qkv, dqkv, nullptr, 0.0f);
            if (!first) { q.a_ss = ss_a; q.a_ss_parts = ssp; }
            L.qkv = make_gemm_plan(q);
            GemmDesc o = dense(att, dm, lw.wo, dm, lw.bo, GEMM_ACT_NONE, y, dm, x, desc.deepnorm_alpha);
            if (!first) { o.res_ss = ss_a; o.res_ss_parts = ssp; o.res_gain = layers[l - 1].n2; }
            L.out_proj = make_gemm_plan(o);
            GemmDesc f1 = dense(qkv, dm, lw.w1_e4m3, 2 * ff, nullptr, GEMM_ACT_SWIGLU, hid, ff, nullptr, 0.0f);
            f1.in_type = GEMM_E4M3;
            f1.out_type = GEMM_E4M3;
            L.fc1 = make_gemm_plan(f1);
            GemmDesc f2 = dense(hid, ff, lw.w2_e4m3, dm, nullptr, GEMM_ACT_NONE, x, dm, att, desc.deepnorm_alpha);
            f2.in_type = GEMM_E4M3;
            f2.out_ss = ss_a;
            L.fc2 = make_gemm_plan(f2);
        } else if (fold_norm) {
            // x holds u_prev (un-normalised, ss_a) except before layer 0, y will hold u_mid (ss_b)
            const bool first = l == 0;
            GemmDesc q = dense(x, dm, lw.wqkv, dqkv, nullptr, GEMM_ACT_ROPE, qkv, dqkv, nullptr, 0.0f);
            if (!first) { q.a_ss = ss_a; q.a_ss_parts = ssp; }
            L.qkv = make_gemm_plan(q);
            GemmDesc o = dense(att, dm, lw.wo, dm, lw.bo, GEMM_ACT_NONE, y, dm, x, desc.deepnorm_alpha);
            if (!first) { o.res_ss = ss_a; o.res_ss_parts = ssp; o.res_gain = layers[l - 1].n2; }
            o.out_ss = ss_b;
            L.out_proj = make_gemm_plan(o);
            GemmDesc f1 = dense(y, dm, lw.w1, 2 * ff, nullptr, GEMM_ACT_SWIGLU, hid, ff, nullptr, 0.0f);
            f1.a_ss = ss_b; f1.a_ss_parts = ssp;
            L.fc1 = make_gemm_plan(f1);
            GemmDesc f2 = dense(hid, ff, lw.w2, dm, nullptr, GEMM_ACT_NONE, x, dm, y, desc.deepnorm_alpha);
            f2.res_ss = ss_b; f2.res_ss_parts = ssp; f2.res_gain = lw.n1;
            f2.out_ss = ss_a;
            L.fc2 = make_gemm_plan(f2);
        } else {
            L.qkv = make_gemm_plan(dense(x, dm, lw.wqkv, dqkv, nullptr, GEMM_ACT_ROPE, qkv, dqkv, nullptr, 0.0f));
            L.out_proj = make_gemm_plan(dense(att, dm, lw.wo, dm, lw.bo, GEMM_ACT_NONE, y, dm, x, desc.deepnorm_alpha));
            L.fc1 = make_gemm_plan(dense(x, dm, lw.w1, 2 * ff, nullptr, GEMM_ACT_SWIGLU, hid, ff, nullptr, 0.0f));
            L.fc2 = make_gemm_plan(dense(hid, ff, lw.w2, dm, nullptr, GEMM_ACT_NONE, y, dm, x, desc.deepnorm_alpha));
        }
        L.n1 = lw.n1;
        L.n2 = lw.n2;
        plan->layers.push_back(L);
    }
    {
        GemmDesc u = dense(x, dm, wu, desc.upsample_scale * dm, bu, GEMM_ACT_NONE, ups, desc.upsample_scale * dm, nullptr, 0.0f);
        if (fold_norm && desc.depth > 0) { u.a_ss = ss_a; u.a_ss_parts = ssp; }
        plan->upsample = make_gemm_plan(u);
    }
    {
        GemmDesc g{};
        g.a = ups;
        g.batches = 1;
        g.rows_per_batch = (int)(rows * desc.upsample_scale);
        g.a_row_stride = dm;
        g.a_batch_stride = (int64_t)rows * desc.upsample_scale * dm;
        g.w = wc;
        g.N = desc.outsize;
        g.K = dm;
        g.act = GEMM_ACT_NONE;
        g.out = scores;
        g.out_m1 = 1;
        g.out_s0 = desc.outsize;
        plan->crf = make_gemm_plan(g);
    }
    plan->qkv_map = make_tmap_2d(qkv, (uint64_t)dqkv, (uint64_t)rows, (uint64_t)dqkv * 2, ATT_D, AT_BQ);
    plan->attn_tc_p = AttnTcParams{att, N, T, desc.nhead, desc.attn_window_upper, desc.attn_window_lower};
    plan->x = x;
    plan->y = y;
    plan->rows = rows;
    plan->N = N;
    plan->T = T;
    plan->H = desc.nhead;
    plan->norm_dim = dm;
    plan->fold_norm = fold_norm;
    plan->fp8 = fp8;
    plan->i8 = i8;
    plan->norm_out = att;
    plan->norm_out8 = reinterpret_cast<uint8_t*>(qkv);
    plan->x8 = x8;
    plan->x_inv = x_inv;
    plan->n_launches = 1 + (desc.num_convs - 1) + (i8 ? 1 : 0) + desc.depth * (i8 ? 7 : fp8 ? 6 : fold_norm ? 5 : 7) + 2;
    if (const char* dbg = std::getenv("B200_DEBUG_TX_LAUNCHES")) {   // debug: stop after k launches (tests/test_tx_layers_gpu.py)
        const int k = std::atoi(dbg);
        if (k >= 0 && k < plan->n_launches) plan->stop_after = k;
    }
    return plan;
}

void TxPlan::run(cudaStream_t stream, ProfileSink* prof) {
    if (stop_after == 0) return;
    // done(name) after every launch: marks it for the profile and says whether B200_DEBUG_TX_LAUNCHES stops the plan there
    int launched = 0;
    auto done = [&](const char* name) {
        if (prof) prof->mark(name, stream);
        if (++launched != stop_after) return false;
        B200_CUDA(cudaGetLastError());
        return true;
    };
    {
        NvtxRange r("Conv");
        const long long total = (long long)conv1.N * conv1.T * (conv1.C1 / 8);
        tx_conv1_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(conv1);
        if (done("tx_conv1")) return;
        for (auto& c : convs) {
            run_gemm(c, stream);
            if (done("tx_conv_gemm")) return;
        }
    }
    const unsigned norm_grid = (unsigned)((rows + 7) / 8);
    if (i8) {
        NvtxRange r("Quantise I8");
        quantize_i8_kernel<<<norm_grid, 256, 0, stream>>>(x, rows, norm_dim, x8, x_inv);
        if (done("quantize_i8")) return;
    }
    {
        NvtxRange enc("TransEnc");
        for (auto& L : layers) {
            NvtxRange layer("TxLayerKoiTiled");
            {
                NvtxRange r("QKV+ROTE");
                run_gemm(L.qkv, stream);
                if (done("qkv_gemm")) return;
            }
            {
                NvtxRange r("MEA");
                launch_attention(qkv_map, attn_tc_p, stream);
                if (done("tx_attention")) return;
            }
            {
                NvtxRange r("OUTP");
                run_gemm(L.out_proj, stream);
                if (done("out_proj_gemm")) return;
            }
            if (fp8) {
                NvtxRange r("LNORM1");
                rmsnorm_kernel<<<norm_grid, 256, 0, stream>>>(y, norm_out, L.n1, rows, norm_dim, norm_out8, nullptr, nullptr);
                if (done("rmsnorm_e4m3")) return;
            } else if (!fold_norm) {
                NvtxRange r("LNORM1");
                rmsnorm_kernel<<<norm_grid, 256, 0, stream>>>(y, x, L.n1, rows, norm_dim, nullptr, nullptr, nullptr);
                if (done("rmsnorm")) return;
            }
            {
                NvtxRange r("FC1+SILU");
                run_gemm(L.fc1, stream);
                if (done("fc1_swiglu_gemm")) return;
            }
            {
                NvtxRange r("FC2");
                run_gemm(L.fc2, stream);
                if (done("fc2_gemm")) return;
            }
            if (!fold_norm) {
                NvtxRange r("LNORM2");
                rmsnorm_kernel<<<norm_grid, 256, 0, stream>>>(y, x, L.n2, rows, norm_dim, nullptr, x8, x_inv);   // x8: int8_qkv only
                if (done(i8 ? "rmsnorm_i8" : "rmsnorm")) return;
            }
        }
    }
    {
        NvtxRange r("TransDec");
        run_gemm(upsample, stream);
        if (done("upsample_gemm")) return;
    }
    {
        NvtxRange r("CRF");
        run_gemm(crf, stream);
        done("crf_gemm");
    }
    B200_CUDA(cudaGetLastError());
}

}  // namespace

std::unique_ptr<Model> make_tx_model(const b200_model_desc& desc, const b200_tensor* tensors, int n) {
    return std::make_unique<TxModel>(desc, tensors, n);
}

// ------------------------------------------------------------------------------------------------
// test hook: host buffers in, host buffer out, the model's attention launch in between
// ------------------------------------------------------------------------------------------------
// ------------------------------------------------------------------------------------------------
// host-side rounding of the fp8_ffn weights
// ------------------------------------------------------------------------------------------------
uint16_t f16_bits(float v) {
    const __half h = __float2half_rn(v);
    uint16_t b;
    std::memcpy(&b, &h, 2);
    return b;
}

static float f16_value(uint16_t b) {
    __half h;
    std::memcpy(&h, &b, 2);
    return __half2float(h);
}

uint16_t remove_bits_f16(uint16_t b, int bits) {
    if (bits <= 0) return b;
    // the reference's integer trick on the int16 view: add half an ulp of the kept mantissa, clear the low bits.  Carries
    // run into the exponent, so the values next to +-65504 become +-inf (the reference's own TODO, TxModules.cpp:107).
    return (uint16_t)((b + (1u << (bits - 1))) & (0xffffu & ~((1u << bits) - 1u)));
}

std::vector<float> fp16_remove_bits(const float* v, size_t n, int bits) {
    std::vector<float> out(n);
    for (size_t i = 0; i < n; ++i) out[i] = f16_value(remove_bits_f16(f16_bits(v[i]), bits));
    return out;
}

uint8_t e4m3_from_f16_bits(uint16_t b) {
    // torch's float -> float8_e4m3fn cast of the fp16 value: round to nearest even; |x| >= 480 (after rounding beyond 448),
    // inf and NaN give NaN (0x7f with the sign), there is no saturation
    const float f = f16_value(b);
    uint32_t u;
    std::memcpy(&u, &f, 4);
    const uint8_t sign = (uint8_t)((b >> 8) & 0x80u);   // from the fp16 bits: the host fp16 -> float conversion drops a NaN's sign
    u &= 0x7fffffffu;
    if (u >= 0x43f00000u) return sign | 0x7f;                              // 480
    if (u < 0x3c800000u) return sign | (uint8_t)std::nearbyint(std::fabs(f) * 512.0f);   // below 2^-6: multiples of 2^-9
    uint32_t keep = u >> 20;                                                 // sign-less exponent and 3 mantissa bits
    const uint32_t rest = u & 0xfffffu;
    if (rest > 0x80000u || (rest == 0x80000u && (keep & 1u))) ++keep;
    return sign | (uint8_t)(keep - ((127u - 7u) << 3));
}

void test_quantize_act_rows_host(int device, const uint16_t* f16, int rows, int cols, int8_t* q, float* inv) {
    if (rows < 1 || cols < 128 || cols % 128 != 0 || (long long)rows * cols >= (1LL << 40)) {
        throw std::invalid_argument("test_quantize_act_rows: rows >= 1 and cols a positive multiple of 128");
    }
    require_sm90(device);
    const size_t n = (size_t)rows * cols;
    __half* d_in = nullptr;
    int8_t* d_q = nullptr;
    float* d_inv = nullptr;
    Arena arena;
    arena.allocate([&](Bump& b) {
        d_in = b.take<__half>(n * 2);
        d_q = b.take<int8_t>(n);
        d_inv = b.take<float>((size_t)rows * 4);
    });
    B200_CUDA(cudaMemcpy(d_in, f16, n * 2, cudaMemcpyHostToDevice));
    quantize_i8_kernel<<<(unsigned)((rows + 7) / 8), 256>>>(d_in, rows, cols, d_q, d_inv);
    B200_CUDA(cudaGetLastError());
    B200_CUDA(cudaDeviceSynchronize());
    B200_CUDA(cudaMemcpy(q, d_q, n, cudaMemcpyDeviceToHost));
    B200_CUDA(cudaMemcpy(inv, d_inv, (size_t)rows * 4, cudaMemcpyDeviceToHost));
}

void test_attention_host(int device, const uint16_t* qkv, int N, int T, int H, int win_upper, int win_lower, uint16_t* out) {
    if (N < 1 || T < 1 || H < 1 || H > 65535 || N > 65535) throw std::invalid_argument("test_attention: bad N, T or H");
    check_attention_window(win_upper, win_lower);
    require_sm90(device);
    const size_t rows = (size_t)N * T, qkv_b = rows * 3 * H * ATT_D * 2, out_b = rows * H * ATT_D * 2;
    __half *d_qkv = nullptr, *d_out = nullptr;
    Arena arena;
    arena.allocate([&](Bump& b) {
        d_qkv = b.take<__half>(qkv_b);
        d_out = b.take<__half>(out_b);
    });
    B200_CUDA(cudaMemcpy(d_qkv, qkv, qkv_b, cudaMemcpyHostToDevice));
    B200_CUDA(cudaMemset(d_out, 0, out_b));
    const CUtensorMap map = make_tmap_2d(d_qkv, (uint64_t)3 * H * ATT_D, (uint64_t)rows, (uint64_t)3 * H * ATT_D * 2, ATT_D, AT_BQ);
    launch_attention(map, AttnTcParams{d_out, N, T, H, win_upper, win_lower}, nullptr);
    B200_CUDA(cudaGetLastError());
    B200_CUDA(cudaDeviceSynchronize());
    B200_CUDA(cudaMemcpy(out, d_out, out_b, cudaMemcpyDeviceToHost));
}

}  // namespace b200
