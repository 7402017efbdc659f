// Conv -> LSTM -> linear CRF forward (fast / hac models) for sm_90a.
//
// Replaces, for the CUDA path of dorado/basecall/model/CRFModel.cpp:69-115:
//   ConvStack layers 1,2   host_convolution_f16              dorado/nn/ConvStack.cpp:216-232  -> conv12_tc_kernel (conv2 on
//                                                                                         mma.sync; v5 shapes), conv12_kernel (FMA pipe)
//   ConvStack layer 3      host_linear "cutlass conv"        dorado/nn/ConvStack.cpp:236-275  -> gemm.cu
//   LSTMStack              host_cutlass_lstm/host_small_lstm dorado/nn/LSTMStack.cpp:127-238 -> gx GEMM + lstm_rec_kernel
//   LinearCRF              host_linear                       dorado/nn/CRFModules.cpp:49-122   -> gemm.cu
// Semantics are those of the CPU modules (ConvStack.cpp:146-163, LSTMStack.cpp:29-41, CRFModules.cpp:24-34).
//
// Activation layouts in HBM (fp16):
//   signal  [N][T_in]
//   x2      [N][T_in + 2*pad3 + 8][16]      conv2 output, NTC, zero rows = conv3's padding (+ K padding)
//   seq     [T_out][N][C]                   time-major LSTM buffer, updated in place by every layer
//   scores  [N][T_out][outsize]
#include "engine.h"
#include "gemm.h"
#include "nvtx.h"
#include "tc.cuh"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include <cooperative_groups.h>

namespace cg = cooperative_groups;

namespace b200 {

namespace {

// ------------------------------------------------------------------------------------------------
// conv1 (1 -> C1, w1) + conv2 (C1 -> 16, w2), both stride 1, fused; fp32 math, fp16 NTC output.
// ------------------------------------------------------------------------------------------------
constexpr int CONV_TT = 256;  // output samples per CTA
constexpr int MAXW = 9;

struct Conv12Params {
    const __half* x;  // [N][T]
    __half* out;      // [N][T_pad][16], row r <-> sample r - front_pad
    const float* w;   // packed: w1 [c1][w1] | b1 [16] | w2 [k][ci][co] (16x16 per tap) | b2 [16]
    int N, T, T_pad, front_pad;
    int c1, w1, w2, act1, act2;
    const int32_t* lens;  // optional per-chunk length in samples (variable chunk sizes): the chunk is zero beyond it
    int* tile_counter;    // conv12_tc_kernel: next tile to hand out (zeroed on the stream before every launch)
};

constexpr int CONV_W_FLOATS = 16 * MAXW + 16 + MAXW * 16 * 16 + 16;

// swish(v) = v / (1 + e^-v), optionally capped at 3.5, or tanh(v) = 1 - 2 / (e^{2v} + 1): one branch-free path (ex2, rcp, select,
// fma, min) whose constants are picked once per thread -- a switch on the run-time activation would be if-converted and every
// element would pay for every variant's transcendentals
struct ConvAct {
    float k, cap;
    bool is_tanh;
};
__device__ __forceinline__ ConvAct conv_act_coef(int act) {
    ConvAct c;
    c.is_tanh = act != B200_ACT_SWISH && act != B200_ACT_SWISH_CLAMP;
    c.k = c.is_tanh ? 2.885390081777927f : -1.4426950408889634f;
    c.cap = act == B200_ACT_SWISH_CLAMP ? 3.5f : __int_as_float(0x7f800000);
    return c;
}
__device__ __forceinline__ float conv_act(float v, const ConvAct& c) {
    const float r = rcp_approx(1.0f + ex2_approx(c.k * v));
    return fminf(c.is_tanh ? fmaf(-2.0f, r, 1.0f) : v * r, c.cap);
}

__global__ void __launch_bounds__(CONV_TT) conv12_kernel(const Conv12Params p) {
    const ConvAct a1 = conv_act_coef(p.act1), a2 = conv_act_coef(p.act2);
    const int n = blockIdx.y;
    const int t0 = blockIdx.x * CONV_TT;
    const int p1 = p.w1 / 2, p2 = p.w2 / 2;
    const int L = p.lens ? min(p.T, __ldg(p.lens + n)) : p.T;  // samples of this chunk (zero padding starts at L)
    constexpr int Y1P = CONV_TT + 2 * MAXW;  // channel-major pitch: consecutive threads -> consecutive banks
    __shared__ float xs[CONV_TT + 4 * MAXW];
    __shared__ float y1[16 * Y1P];
    __shared__ __align__(16) float ws[CONV_W_FLOATS];
    const float* s_w1 = ws;
    const float* s_b1 = ws + 16 * MAXW;
    const float* s_w2 = s_b1 + 16;
    const float* s_b2 = s_w2 + MAXW * 16 * 16;
    for (int i = threadIdx.x; i < CONV_W_FLOATS; i += CONV_TT) ws[i] = __ldg(p.w + i);
    const int nx = CONV_TT + 2 * (p1 + p2);
    for (int i = threadIdx.x; i < nx; i += CONV_TT) {
        const int t = t0 - p1 - p2 + i;
        xs[i] = (t >= 0 && t < L) ? __half2float(p.x[(size_t)n * p.T + t]) : 0.0f;
    }
    __syncthreads();
    const int n1 = CONV_TT + 2 * p2;
    for (int i = threadIdx.x; i < n1; i += CONV_TT) {
        const int t = t0 - p2 + i;  // conv1 output position
        const bool inside = t >= 0 && t < L;
        for (int c = 0; c < p.c1; ++c) {
            float acc = s_b1[c];
            for (int k = 0; k < p.w1; ++k) acc += s_w1[c * p.w1 + k] * xs[i + k];
            y1[c * Y1P + i] = inside ? conv_act(acc, a1) : 0.0f;  // conv2 zero-pads conv1's *output*
        }
    }
    __syncthreads();
    const int t = t0 + threadIdx.x;
    if (t < p.T) {
        float acc[16];
#pragma unroll
        for (int co = 0; co < 16; ++co) acc[co] = s_b2[co];
        for (int k = 0; k < p.w2; ++k) {
            for (int ci = 0; ci < p.c1; ++ci) {
                const float v = y1[ci * Y1P + threadIdx.x + k];
                const float4* w = reinterpret_cast<const float4*>(&s_w2[(k * 16 + ci) * 16]);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float4 wv = w[q];
                    acc[4 * q + 0] += v * wv.x;
                    acc[4 * q + 1] += v * wv.y;
                    acc[4 * q + 2] += v * wv.z;
                    acc[4 * q + 3] += v * wv.w;
                }
            }
        }
        __half2 h[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) h[j] = __floats2half2_rn(conv_act(acc[2 * j], a2), conv_act(acc[2 * j + 1], a2));
        if (t >= L) {  // beyond a short chunk's end: the next convolution's zero padding
#pragma unroll
            for (int j = 0; j < 8; ++j) h[j] = __floats2half2_rn(0.0f, 0.0f);
        }
        uint4* dst = reinterpret_cast<uint4*>(p.out + ((size_t)n * p.T_pad + p.front_pad + t) * 16);
        dst[0] = *reinterpret_cast<uint4*>(&h[0]);
        dst[1] = *reinterpret_cast<uint4*>(&h[4]);
    }
}

// ------------------------------------------------------------------------------------------------
// conv1 + conv2 with conv2 on the tensor cores (the v5 shape: conv1 1 -> 16, conv2 16 -> 16 with 5 taps).
//
// conv2 is 1280 of the 1360 multiply-adds per sample; on the FMA pipe (conv12_kernel above) that is 1.4e10 FLOP per batch of
// 512 x 9996 samples for a kernel that should be bound by HBM (2 B in, 32 B out per sample).  Here a tile of 128 output
// samples is one M = 128, N = 16, K = 80 contraction on mma.sync:
//   * conv1 (+ activation) runs on the FMA pipe, one thread per conv1 position, and its 16 channels are rounded to fp16
//     (every activation tensor between layers is fp16, as in the reference's CUDA path);
//   * the A operand is conv2's im2col tile built directly in shared memory in a 128-byte-swizzled K-major layout:
//     K index = tap * 16 + channel, so the 32 bytes of conv1 position j go to row j - tap, 16-byte chunks 2 tap and 2 tap + 1
//     (five 2 x 16 B stores per thread; the XOR swizzle keeps the eight rows of an ldmatrix phase on distinct banks);
//   * B = the conv2 weights [16][80] fp16 in the same layout, written once per CTA and held in registers as mma fragments;
//   * warps 0-3 each contract 32 rows (2 x 2 m16n8k16 tiles, 5 K steps), add the bias, apply the activation and store
//     the samples' 16 fp16 channels.
// The phases of a tile are separated by CTA barriers; several CTAs share an SM and hide each other's barriers.  The grid
// is persistent and takes tiles from a counter.
// ------------------------------------------------------------------------------------------------
constexpr int C12_TILE = 128;
// warps 0-3: conv1 producers, MMA and epilogue (32 rows each); warp 4: conv1 tail positions; warp 5 idle
constexpr int C12_THREADS = 192;
constexpr int C12_SMEM = 2 * 16384 + 2 * 2048 + 1024;  // A (2 k-blocks of 128 rows x 128 B), B (2 k-blocks of 16 rows), alignment slack

__global__ void __launch_bounds__(C12_THREADS, 4) conv12_tc_kernel(const Conv12Params p, int tiles_per_chunk, int num_tiles) {
    extern __shared__ __align__(1024) uint8_t c12_smem_raw[];
    uint8_t* smem = c12_smem_raw + ((1024u - (tc::smem_u32(c12_smem_raw) & 1023u)) & 1023u);
    uint8_t* a_tile = smem;               // [2][128 rows][128 B]
    uint8_t* b_tile = smem + 2 * 16384;   // [2][16 rows][128 B]
    __shared__ float xs[C12_TILE + 4 + 2 * MAXW];
    __shared__ float s_w1[16 * MAXW], s_b1[16], s_b2[16];
    __shared__ int s_tile;
    const ConvAct a1 = conv_act_coef(p.act1), a2 = conv_act_coef(p.act2);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int p1 = p.w1 / 2;
    constexpr int p2 = 2;

    // ---- once per CTA: conv1 weights / biases, conv2 weights as the fp16 B operand
    for (int i = tid; i < 16 * MAXW; i += C12_THREADS) s_w1[i] = __ldg(p.w + i);
    if (tid < 16) {
        s_b1[tid] = __ldg(p.w + 16 * MAXW + tid);
        s_b2[tid] = __ldg(p.w + 16 * MAXW + 16 + MAXW * 16 * 16 + tid);
    }
    for (int i = tid; i < 2 * 2048 / 16; i += C12_THREADS) reinterpret_cast<uint4*>(b_tile)[i] = make_uint4(0, 0, 0, 0);
    __syncthreads();
    {
        const float* w2 = p.w + 16 * MAXW + 16;  // [tap][ci][co]
        for (int i = tid; i < 5 * 16 * 16; i += C12_THREADS) {
            const int co = i & 15, ci = (i >> 4) & 15, tap = i >> 8;
            const int c = (tap * 2 + (ci >> 3)) & 7, kb = tap >> 2;
            *reinterpret_cast<__half*>(b_tile + kb * 2048 + tc::sw128_offset(co, c) + (ci & 7) * 2) =
                    __float2half_rn(__ldg(w2 + (tap * 16 + ci) * 16 + co));
        }
    }
    __syncthreads();
    // B fragments of the five K steps: matrix q of ldmatrix.x4 = (n tile q / 2, k half q % 2)
    uint32_t bfrag[5][4];
    if (warp < 4) {
        const int q = lane >> 3, r = lane & 7;
#pragma unroll
        for (int tap = 0; tap < 5; ++tap) {
            const int chunk = 2 * tap + (q & 1);
            tc::ldmatrix_x4(bfrag[tap], tc::smem_u32(b_tile + (chunk >> 3) * 2048 + tc::sw128_offset((q >> 1) * 8 + r, chunk & 7)));
        }
    }

    for (;;) {
        __syncthreads();  // the previous tile's MMAs have read A: it may be overwritten
        if (tid == 0) s_tile = atomicAdd(p.tile_counter, 1);
        __syncthreads();
        const int tile = s_tile;
        if (tile >= num_tiles) break;
        const int n = tile / tiles_per_chunk;
        const int t0 = (tile - n * tiles_per_chunk) * C12_TILE;
        const int L = p.lens ? min(p.T, __ldg(p.lens + n)) : p.T;  // samples of this chunk (zero padding starts at L)
        // ---- signal window: xs[i] <-> sample t0 - p2 - p1 + i
        if (tid < C12_TILE + 2 * (p1 + p2)) {
            const int t = t0 - p2 - p1 + tid;
            xs[tid] = (t >= 0 && t < L) ? __half2float(p.x[(size_t)n * p.T + t]) : 0.0f;
        }
        __syncthreads();
        // ---- conv1 at position j <-> sample t0 - p2 + j, scattered into the im2col rows j - tap
        if (tid < C12_TILE + 2 * p2) {
            const int j = tid;
            const int t = t0 - p2 + j;
            const bool inside = t >= 0 && t < L;  // conv2 zero-pads conv1's *output*
            float xv[MAXW];
#pragma unroll
            for (int k = 0; k < MAXW; ++k) xv[k] = k < p.w1 ? xs[j + k] : 0.0f;
            __half2 h[8];
#pragma unroll
            for (int c2 = 0; c2 < 8; ++c2) {
                float acc0 = s_b1[2 * c2], acc1 = s_b1[2 * c2 + 1];
#pragma unroll
                for (int k = 0; k < MAXW; ++k) {
                    if (k < p.w1) {
                        acc0 = fmaf(s_w1[(2 * c2) * p.w1 + k], xv[k], acc0);
                        acc1 = fmaf(s_w1[(2 * c2 + 1) * p.w1 + k], xv[k], acc1);
                    }
                }
                h[c2] = inside ? __floats2half2_rn(conv_act(acc0, a1), conv_act(acc1, a1)) : __floats2half2_rn(0.0f, 0.0f);
            }
            const uint4 lo = *reinterpret_cast<const uint4*>(&h[0]), hi = *reinterpret_cast<const uint4*>(&h[4]);
#pragma unroll
            for (int tap = 0; tap < 5; ++tap) {
                const int i = j - tap;
                if (i >= 0 && i < C12_TILE) {
                    uint8_t* base = a_tile + (tap >> 2) * 16384;
                    const int c = (tap * 2) & 7;
                    *reinterpret_cast<uint4*>(base + tc::sw128_offset(i, c)) = lo;
                    *reinterpret_cast<uint4*>(base + tc::sw128_offset(i, c + 1)) = hi;
                }
            }
        }
        __syncthreads();
        // ---- conv2: warp w contracts rows 32 w .. 32 w + 31, thread = fragment rows lane / 4 (+ 8), channels 2 (lane % 4) (+ 1, + 8)
        if (warp < 4) {
            float acc[2][2][4];
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                for (int nt = 0; nt < 2; ++nt)
#pragma unroll
                    for (int e = 0; e < 4; ++e) acc[mt][nt][e] = 0.0f;
            const int q = lane >> 3, r = lane & 7;
#pragma unroll
            for (int tap = 0; tap < 5; ++tap) {
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) {
                    // matrix q of ldmatrix.x4 = (row half q % 2, k half q / 2): the a0..a3 order of m16n8k16
                    const int row = warp * 32 + mt * 16 + (q & 1) * 8 + r, chunk = 2 * tap + (q >> 1);
                    uint32_t a[4];
                    tc::ldmatrix_x4(a, tc::smem_u32(a_tile + (chunk >> 3) * 16384 + tc::sw128_offset(row, chunk & 7)));
                    tc::mma_f16_16816(acc[mt][0], a, bfrag[tap][0], bfrag[tap][1]);
                    tc::mma_f16_16816(acc[mt][1], a, bfrag[tap][2], bfrag[tap][3]);
                }
            }
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    const int t = t0 + warp * 32 + mt * 16 + (lane >> 2) + 8 * hh;
                    if (t >= p.T) continue;
                    __half* dst = p.out + ((size_t)n * p.T_pad + p.front_pad + t) * 16;
#pragma unroll
                    for (int nt = 0; nt < 2; ++nt) {
                        const int co = nt * 8 + 2 * (lane & 3);
                        __half2 o = __floats2half2_rn(conv_act(acc[mt][nt][2 * hh] + s_b2[co], a2),
                                                      conv_act(acc[mt][nt][2 * hh + 1] + s_b2[co + 1], a2));
                        if (t >= L) o = __floats2half2_rn(0.0f, 0.0f);  // beyond a short chunk's end: the next convolution's zero padding
                        *reinterpret_cast<__half2*>(dst + co) = o;
                    }
                }
            }
        }
    }
}

// Gate activations on one MUFU.TANH each: sigmoid(v) = 0.5 tanh(0.5 v) + 0.5 (am = 1), tanh(v) (am = 2); FMUL, MUFU.TANH, FFMA.
// tanh.approx.f32 is good to ~2^-11 -- the rounding h_t gets anyway when it is stored as fp16, and the gates saturate and
// contract the error.  The same substitution in the swish of the convolutions was rejected, see common.cuh.
// -DB200_LSTM_EX2_RCP restores the two-MUFU form (ex2 + rcp).
#ifndef B200_LSTM_EX2_RCP
__device__ __forceinline__ float gate_act(float v, float am) {
    const float s = 0.5f * am;
    return fmaf(tanh_mufu(v * s), s, 1.0f - s);
}
#else
__device__ __forceinline__ float gate_act(float v, float am) {
    float e, r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(v * (am * 1.4426950408889634f)));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(e + 1.0f));
    return fmaf(-am, r, 1.0f);
}
#endif
__device__ __forceinline__ float tanh_f(float v) { return gate_act(v, 2.0f); }

// ------------------------------------------------------------------------------------------------
// LSTM layer = hoisted x-projection + recurrence.
//
// The x_t half of the gate pre-activations does not depend on the recurrence, so it is one large wgmma GEMM per layer
// (gemm.cu) that writes gx[t][chunk][4C] (fp16, b_ih + b_hh included, PyTorch gate order i | f | g | o).
//
// Recurrence (lstm_rec_kernel): a thread-block cluster of CL CTAs owns NB chunks; CTA `rank` owns hidden units
// [rank * U, rank * U + U), U = C / CL, i.e. 4U gate rows of W_hh.  Those rows live in REGISTERS for the whole sequence, as
// mma.sync A fragments: warp w holds gate rows 16 w .. 16 w + 15 for all of K = C (C / 16 x 4 registers per thread).  A
// step is
//     G[4U][NB] = W_hh[rows of this CTA] h_{t-1}      mma.sync m16n8k16, B fragments by ldmatrix from this CTA's copy of h
//     gates, cell update, h_t (fp16)                    thread = a pair of adjacent units x one chunk, cell state in registers
//     h_t -> every CTA's copy of h (distributed shared memory) and to the sequence buffer, one cluster barrier
// The step is a latency chain (MMA -> barrier -> gate math -> all-gather -> barrier) rather than a throughput problem:
// mma.sync on register-resident weights keeps that chain short, where wgmma would add its asynchronous hand-offs and a
// 64-row granularity to every step.  h is double-buffered, so one cluster barrier per step orders both the all-gather of
// h_t before the MMAs of step t+1 and the reads of h_{t-1} before its buffer is overwritten at step t+1.
// C = 96 runs as a cluster of one CTA (all 384 gate rows in one CTA); C = 192 and 384 split over 4 and 8 CTAs.
// ------------------------------------------------------------------------------------------------
struct LstmRecParams {
    __half* seq;          // [T][N][C] output h (in place over the layer input, which gx has consumed)
    const __half* gx;     // [T][N][4C]
    const __half* w_hh;   // [4C][C], PyTorch row order
    int T, N, reverse;
    const int32_t* lens;  // optional per-chunk length in samples (variable chunk sizes); stride = samples per step
    int stride;
};

// CTAs per cluster for a hidden size: the CTA's W_hh rows (4 C / CL x C fp16) must fit its registers
__host__ __device__ constexpr int rec_cluster(int C) { return C <= 96 ? 1 : C <= 192 ? 4 : 8; }

template <int C, int CL, int NB>
struct RecCfg {
    static constexpr int U = C / CL;              // hidden units per CTA
    static constexpr int MT = 4 * U / 16;         // m16 tiles of gate rows = warps
    static constexpr int THREADS = 32 * MT;
    static constexpr int KS = C / 16;             // K steps
    static constexpr int NT = NB / 8;             // n8 tiles of chunks
    static constexpr int HS = C + 8;              // row stride of h (fp16): the 8 rows of an ldmatrix phase on distinct banks
    static constexpr int GS = NB + 4;             // row stride of the gate pre-activations (fp32)
    static constexpr int PAIRS = U / 2 * NB / THREADS;   // (unit pair, chunk) cells per thread
    // gx is loaded ahead of the MMAs when it fits the registers; with 4 cell pairs per thread (64 chunks per cluster) the
    // 16 extra registers would spill, so gx is loaded in the cell loop instead
    static constexpr bool GX_AHEAD = PAIRS <= 2;
    static constexpr size_t SMEM = (size_t)2 * NB * HS * 2 + (size_t)4 * U * GS * 4;
    static_assert(C % CL == 0 && U % 4 == 0 && NT % 2 == 0 && PAIRS >= 1 && (U / 2 * NB) % THREADS == 0, "recurrence shape");
    static_assert(THREADS <= 1024 && CL <= 8, "block / cluster size");
};

template <int C, int CL, int NB>
__global__ void __launch_bounds__(RecCfg<C, CL, NB>::THREADS, 1) lstm_rec_kernel(const LstmRecParams p) {
    using Cfg = RecCfg<C, CL, NB>;
    constexpr int U = Cfg::U, KS = Cfg::KS, NT = Cfg::NT, HS = Cfg::HS, GS = Cfg::GS, PAIRS = Cfg::PAIRS;
    constexpr bool GX_AHEAD = Cfg::GX_AHEAD;
    extern __shared__ __align__(16) uint8_t smem_raw[];
    __half* h_s = reinterpret_cast<__half*>(smem_raw);                      // [2][NB][HS]  this CTA's copy of h
    float* g_s = reinterpret_cast<float*>(smem_raw + (size_t)2 * NB * HS * 2);  // [4U][GS]
    __shared__ int len_s[NB];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    cg::cluster_group cluster = cg::this_cluster();
    const int rank = CL > 1 ? (int)cluster.block_rank() : 0;
    const int n0 = (int)(blockIdx.x / CL) * NB;
    if (threadIdx.x < NB) len_s[threadIdx.x] = p.lens ? min(p.T, __ldg(p.lens + n0 + threadIdx.x) / p.stride) : p.T;
    for (int i = threadIdx.x; i < 2 * NB * HS / 8; i += Cfg::THREADS) reinterpret_cast<uint4*>(h_s)[i] = make_uint4(0, 0, 0, 0);

    // A fragments: local gate row r <-> W_hh row (r / U) * C + rank * U + r % U
    uint32_t a[KS][4];
    {
        const int r_lo = warp * 16 + (lane >> 2), r_hi = r_lo + 8;
        const __half* w_lo = p.w_hh + (size_t)((r_lo / U) * C + rank * U + r_lo % U) * C;
        const __half* w_hi = p.w_hh + (size_t)((r_hi / U) * C + rank * U + r_hi % U) * C;
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
            const int col = ks * 16 + 2 * (lane & 3);
            a[ks][0] = __ldg(reinterpret_cast<const unsigned int*>(w_lo + col));
            a[ks][1] = __ldg(reinterpret_cast<const unsigned int*>(w_hi + col));
            a[ks][2] = __ldg(reinterpret_cast<const unsigned int*>(w_lo + col + 8));
            a[ks][3] = __ldg(reinterpret_cast<const unsigned int*>(w_hi + col + 8));
        }
    }
    // cells: pair index q = threadIdx.x + j * THREADS -> units (u, u + 1), u = 2 (q % (U / 2)), chunk q / (U / 2)
    float c_reg[PAIRS][2];
#pragma unroll
    for (int j = 0; j < PAIRS; ++j) c_reg[j][0] = c_reg[j][1] = 0.0f;
    // every CTA of the cluster has zeroed its copy of h before anybody writes h_0 into it
    if constexpr (CL > 1) cluster.sync();
    else __syncthreads();

    int steps = 0;
    for (int i = 0; i < NB; ++i) steps = max(steps, len_s[i]);
    const int qm = lane >> 3, qr = lane & 7;   // ldmatrix: matrix qm = (n tile qm / 2, k half qm % 2), row qr
    for (int s = 0; s < steps; ++s) {
        const int t = p.reverse ? steps - 1 - s : s;
        const int cur = s & 1, nxt = cur ^ 1;
        // gx of this thread's cells: independent of the recurrence, in flight while the MMAs run (GX_AHEAD)
        auto load_gx = [&](int j, __half2* dst) {
            const int q = threadIdx.x + j * Cfg::THREADS;
            const int u = 2 * (q % (U / 2)), n = q / (U / 2);
            const __half* gp = p.gx + ((size_t)t * p.N + n0 + n) * (4 * C) + rank * U + u;
#pragma unroll
            for (int g = 0; g < 4; ++g) dst[g] = *reinterpret_cast<const __half2*>(gp + g * C);
        };
        __half2 gxv[GX_AHEAD ? PAIRS : 1][4];
        if constexpr (GX_AHEAD) {
#pragma unroll
            for (int j = 0; j < PAIRS; ++j) load_gx(j, gxv[j]);
        }
        float acc[NT][4];
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.0f;
        const uint32_t hb = tc::smem_u32(h_s + cur * NB * HS);
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
#pragma unroll
            for (int np = 0; np < NT / 2; ++np) {
                uint32_t b[4];
                const int n = (2 * np + (qm >> 1)) * 8 + qr, k = ks * 16 + (qm & 1) * 8;
                tc::ldmatrix_x4(b, hb + (uint32_t)((n * HS + k) * 2));
                tc::mma_f16_16816(acc[2 * np], a[ks], b[0], b[1]);
                tc::mma_f16_16816(acc[2 * np + 1], a[ks], b[2], b[3]);
            }
        }
        {
            const int r_lo = warp * 16 + (lane >> 2);
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) {
                const int col = nt * 8 + 2 * (lane & 3);
                *reinterpret_cast<float2*>(g_s + r_lo * GS + col) = make_float2(acc[nt][0], acc[nt][1]);
                *reinterpret_cast<float2*>(g_s + (r_lo + 8) * GS + col) = make_float2(acc[nt][2], acc[nt][3]);
            }
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < PAIRS; ++j) {
            const int q = threadIdx.x + j * Cfg::THREADS;
            const int u = 2 * (q % (U / 2)), n = q / (U / 2);
            // outside the chunk (variable chunk sizes) the state is held at zero: a multiplicative mask, not a branch
            const float alive = t < len_s[n] ? 1.0f : 0.0f;
            __half2 gxl[4];
            const __half2* gxj = gxl;
            if constexpr (GX_AHEAD) gxj = gxv[j];
            else load_gx(j, gxl);
            float hv[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                float pre[4];
#pragma unroll
                for (int g = 0; g < 4; ++g) {
                    const float2 x = __half22float2(gxj[g]);
                    pre[g] = g_s[(g * U + u + e) * GS + n] + (e ? x.y : x.x);
                }
                const float ig = gate_act(pre[0], 1.0f), fg = gate_act(pre[1], 1.0f);
                const float gg = gate_act(pre[2], 2.0f), og = gate_act(pre[3], 1.0f);
                const float cs = (fg * c_reg[j][e] + ig * gg) * alive;
                c_reg[j][e] = cs;
                hv[e] = og * tanh_f(cs) * alive;
            }
            const __half2 h2 = __floats2half2_rn(hv[0], hv[1]);
            *reinterpret_cast<__half2*>(p.seq + ((size_t)t * p.N + n0 + n) * C + rank * U + u) = h2;
            __half* h_own = h_s + (nxt * NB + n) * HS + rank * U + u;
            if constexpr (CL > 1) {
#pragma unroll
                for (int r = 0; r < CL; ++r) *reinterpret_cast<__half2*>(cluster.map_shared_rank(h_own, r)) = h2;
            } else {
                *reinterpret_cast<__half2*>(h_own) = h2;
            }
        }
        // h_t has landed in every copy, and every thread is done with h_{t-1} and the gate buffer
        if constexpr (CL > 1) cluster.sync();
        else __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
struct LstmLayerWeights {
    __half* w_ih = nullptr;  // [4C][Cp] (K padded to a multiple of 64), PyTorch row order
    __half* w_hh = nullptr;  // [4C][C]
    float* bias = nullptr;   // [4C] b_ih + b_hh
};

class LstmModel;

class LstmPlan final : public ForwardPlan {
public:
    void run(cudaStream_t stream, ProfileSink* prof) override;
    int launches() const override { return 1 + 1 + num_layers * 2 + num_linear; }
    std::string info() const override {
        return "lstm_rec.ctas=" + std::to_string(rec_ctas) + ";lstm_rec.chunks_per_cluster=" + std::to_string(rec_un);
    }
    void set_chunk_lengths(const int32_t* d_lens) override {
        if (!variable) return;  // the mode exists for the models that run variable chunk sizes only
        conv12.lens = d_lens;
        for (auto& rp : rec_p) rp.lens = d_lens;
    }

    Conv12Params conv12{};
    dim3 conv12_grid;
    bool conv12_tc = false;  // conv2 on the tensor cores (conv12_tc_kernel)
    int conv12_tiles_per_chunk = 0, conv12_tc_grid = 0;
    GemmPlan conv3;
    int debug_layers = -1;  // >= 0: stop after that many LSTM layers (B200_DEBUG_LSTM_LAYERS, read once at plan creation)
    bool variable = false;
    int rec_un = 16;        // chunks per cluster (NB)
    int rec_ctas = 0;
    std::vector<GemmPlan> gx_gemm;
    std::vector<LstmRecParams> rec_p;
    void launch_rec(int l, cudaStream_t stream) const;
    GemmPlan linear1, linear2;
    int num_layers = 0, num_linear = 1;
    const LstmModel* model = nullptr;
};

class LstmModel final : public Model {
public:
    LstmModel(const b200_model_desc& d, const b200_tensor* tensors, int n);
    ~LstmModel() override;
    size_t workspace_bytes(int N, int T_in) const override;
    std::unique_ptr<ForwardPlan> make_plan(int N, int T_in, const __half* signal, __half* scores, void* ws,
                                           size_t ws_bytes) override;
    bool variable_chunk_sizes() const override {
        // FLSTM models never run variable chunk sizes (api/runner_creation.cpp:28)
        return large() && desc.lstm_inner_dim == 0;
    }

    b200_model_desc desc;
    float* conv_w = nullptr;  // packed conv1 / conv2 weights (see Conv12Params::w)
    __half* w3 = nullptr;               // [C][K3p]
    float* b3 = nullptr;
    int K3 = 0, K3p = 0;
    std::vector<LstmLayerWeights> layers;
    __half* wl1 = nullptr;  // [out1][Cp]
    float* bl1 = nullptr;
    __half* wl2 = nullptr;  // decomposition: [outsize][out_features_p]
    int Cp = 0, out1 = 0, out1p = 0;

private:
    int pad3() const { return desc.convs[2].winlen / 2; }
    int t_pad(int T_in) const { return T_in + 2 * pad3() + 8; }
    // lstm_size 96 keeps the reference's fixed-size contract (batch a multiple of 16, no variable chunk sizes); the larger
    // sizes take batches in multiples of 32 and variable chunk sizes
    bool large() const { return desc.lstm_size > 96; }
    int n_pad(int N) const { return large() ? (N + 31) / 32 * 32 : (N + 15) / 16 * 16; }
};

LstmModel::LstmModel(const b200_model_desc& d, const b200_tensor* tensors, int n) : desc(d) {
    if (d.num_convs != 3) throw std::invalid_argument("Expected 3 convolution layers but found: " + std::to_string(d.num_convs));
    const auto &c1 = d.convs[0], &c2 = d.convs[1], &c3 = d.convs[2];
    if (c1.insize != 1 || c1.stride != 1 || c2.stride != 1 || c2.size != 16 || c1.size > 16 || c1.winlen > MAXW ||
        c2.winlen > MAXW || c2.insize != c1.size || c3.insize != 16) {
        throw Unsupported("conv stack shape outside what conv12_kernel implements");
    }
    const int C = d.lstm_size;
    if (C != c3.size) throw std::invalid_argument("last convolution size != lstm_size");
    if (C != 96 && C != 192 && C != 384) {
        // kernels are instantiated for the sizes of the reference's model zoo this engine covers
        throw Unsupported("lstm_size " + std::to_string(C) + " is not supported (96, 192 and 384 are)");
    }

    if (d.lstm_layers < 1 || d.lstm_layers > 8) throw std::invalid_argument("bad lstm_layers");

    // conv1: torch [c1][1][w] -> [c1][w]; conv2: torch [co][ci][k] -> [k][ci][co]
    {
        const auto& tw = find_tensor(tensors, n, "0.conv.weight.tensor");
        const auto& tb = find_tensor(tensors, n, "0.conv.bias.tensor");
        const auto& tw2 = find_tensor(tensors, n, "1.conv.weight.tensor");
        const auto& tb2 = find_tensor(tensors, n, "1.conv.bias.tensor");
        std::vector<float> pk(CONV_W_FLOATS, 0.0f);
        float* w1 = pk.data();
        float* b1 = w1 + 16 * MAXW;
        float* w2 = b1 + 16;
        float* b2 = w2 + MAXW * 16 * 16;
        std::memcpy(w1, tw.data, sizeof(float) * (size_t)c1.size * c1.winlen);
        std::memcpy(b1, tb.data, sizeof(float) * c1.size);
        for (int co = 0; co < 16; ++co)
            for (int ci = 0; ci < c2.insize; ++ci)
                for (int k = 0; k < c2.winlen; ++k)
                    w2[((size_t)k * 16 + ci) * 16 + co] = tw2.data[((size_t)co * c2.insize + ci) * c2.winlen + k];
        std::memcpy(b2, tb2.data, sizeof(float) * 16);
        conv_w = upload_f32(pk);
    }
    // conv3 as GEMM weights: [C][k*16 + ci], K padded to a multiple of 64
    {
        const auto& tw = find_tensor(tensors, n, "2.conv.weight.tensor");
        const auto& tb = find_tensor(tensors, n, "2.conv.bias.tensor");
        K3 = c3.winlen * 16;
        K3p = (K3 + 63) / 64 * 64;
        std::vector<float> w((size_t)C * K3p, 0.0f);
        for (int co = 0; co < C; ++co)
            for (int ci = 0; ci < 16; ++ci)
                for (int k = 0; k < c3.winlen; ++k)
                    w[(size_t)co * K3p + k * 16 + ci] = tw.data[((size_t)co * 16 + ci) * c3.winlen + k];
        w3 = upload_f16(w);
        b3 = upload_f32(std::vector<float>(tb.data, tb.data + C));
    }
    // LSTM layers: W_ih (K padded for the GEMM), W_hh and the summed biases, gate rows in PyTorch order (i | f | g | o)
    for (int l = 0; l < d.lstm_layers; ++l) {
        const std::string pfx = std::to_string(d.num_convs + l + 1) + ".rnn.";
        // plain LSTM: the tensors as they are.  FLSTM (nn/FLSTMStack.cpp:18-25,108-124): gates = up_ih (dn_ih x_t) +
        // up_hh (dn_hh h_{t-1}) + bias, folded once into W = up x dn (double accumulation, rounded to fp32) so that the
        // x-projection GEMM and the recurrence kernel serve both model kinds.
        struct View { const float* data; };
        std::vector<float> folded_ih, folded_hh;
        View wih{}, whh{}, bih{}, bhh{};
        if (d.lstm_inner_dim > 0) {
            const int K = d.lstm_inner_dim;
            auto fold = [&](const char* up_name, const char* dn_name, std::vector<float>& out) {
                const auto& up = find_tensor(tensors, n, pfx + up_name);
                const auto& dn = find_tensor(tensors, n, pfx + dn_name);
                if (up.ndim != 2 || dn.ndim != 2 || up.dims[0] != 4 * C || up.dims[1] != K || dn.dims[0] != K || dn.dims[1] != C) {
                    throw std::invalid_argument("FLSTM tensor " + pfx + up_name + " / " + dn_name + " has the wrong shape");
                }
                out.assign((size_t)4 * C * C, 0.0f);
                std::vector<double> acc((size_t)C);
                for (int r = 0; r < 4 * C; ++r) {
                    std::fill(acc.begin(), acc.end(), 0.0);
                    for (int k = 0; k < K; ++k) {
                        const double u = up.data[(size_t)r * K + k];
                        const float* drow = dn.data + (size_t)k * C;
                        for (int c2 = 0; c2 < C; ++c2) acc[c2] += u * (double)drow[c2];
                    }
                    for (int c2 = 0; c2 < C; ++c2) out[(size_t)r * C + c2] = (float)acc[c2];
                }
            };
            fold("up_weight_ih.tensor", "dn_weight_ih.tensor", folded_ih);
            fold("up_weight_hh.tensor", "dn_weight_hh.tensor", folded_hh);
            wih.data = folded_ih.data();
            whh.data = folded_hh.data();
            bih.data = find_tensor(tensors, n, pfx + "up_bias_ih.tensor").data;
            bhh.data = find_tensor(tensors, n, pfx + "up_bias_hh.tensor").data;
        } else {
            wih.data = find_tensor(tensors, n, pfx + "weight_ih_l0.tensor").data;
            whh.data = find_tensor(tensors, n, pfx + "weight_hh_l0.tensor").data;
            bih.data = find_tensor(tensors, n, pfx + "bias_ih_l0.tensor").data;
            bhh.data = find_tensor(tensors, n, pfx + "bias_hh_l0.tensor").data;
        }
        const int Cp = (C + 63) / 64 * 64;
        std::vector<float> wi((size_t)4 * C * Cp, 0.0f), b((size_t)4 * C);
        for (int r = 0; r < 4 * C; ++r) {
            std::memcpy(&wi[(size_t)r * Cp], &wih.data[(size_t)r * C], sizeof(float) * C);
            b[r] = bih.data[r] + bhh.data[r];
        }
        LstmLayerWeights lw;
        lw.w_ih = upload_f16(wi);
        lw.w_hh = upload_f16(std::vector<float>(whh.data, whh.data + (size_t)4 * C * C));
        lw.bias = upload_f32(b);
        layers.push_back(lw);
    }
    // linear(s)
    {
        const int layer = d.num_convs + d.lstm_layers + 1;
        const auto& tw = find_tensor(tensors, n, std::to_string(layer) + ".linear.weight.tensor");
        out1 = d.out_features > 0 ? d.out_features : d.outsize;
        Cp = (C + 63) / 64 * 64;
        std::vector<float> w((size_t)out1 * Cp, 0.0f);
        for (int o = 0; o < out1; ++o) std::memcpy(&w[(size_t)o * Cp], &tw.data[(size_t)o * C], sizeof(float) * C);
        wl1 = upload_f16(w);
        if (d.linear_bias) {
            const auto& tb = find_tensor(tensors, n, std::to_string(layer) + ".linear.bias.tensor");
            bl1 = upload_f32(std::vector<float>(tb.data, tb.data + out1));
        }
        if (d.out_features > 0) {
            if (out1 % 64 != 0) throw Unsupported("out_features must be a multiple of 64");
            const auto& tw2 = find_tensor(tensors, n, std::to_string(layer + 1) + ".linear.weight.tensor");
            wl2 = upload_f16(std::vector<float>(tw2.data, tw2.data + (size_t)d.outsize * out1));
        }
    }
}

LstmModel::~LstmModel() {
    cudaFree(conv_w);
    cudaFree(w3);
    cudaFree(b3);
    for (auto& l : layers) {
        cudaFree(l.bias);
        cudaFree(l.w_ih);
        cudaFree(l.w_hh);
    }
    cudaFree(wl1);
    cudaFree(bl1);
    cudaFree(wl2);
}

size_t LstmModel::workspace_bytes(int N, int T_in) const {
    const int T_out = T_in / desc.stride;
    const size_t x2 = (size_t)N * t_pad(T_in) * 16 * 2 + 4096;
    const size_t seq = (size_t)(T_out + 1) * n_pad(N) * desc.lstm_size * 2 + 4096;
    const size_t mid = desc.out_features > 0 ? (size_t)T_out * n_pad(N) * desc.out_features * 2 + 4096 : 0;
    const size_t gx = (size_t)T_out * n_pad(N) * 4 * desc.lstm_size * 2 + 4096;
    return x2 + seq + mid + gx + 4096;  // + the tile counter of conv12_tc_kernel
}

std::unique_ptr<ForwardPlan> LstmModel::make_plan(int N, int T_in, const __half* signal, __half* scores, void* ws,
                                                  size_t ws_bytes) {
    const int C = desc.lstm_size;
    const int T_out = T_in / desc.stride;
    const int Np = n_pad(N);
    if (Np != N) {
        // the reference's tensor-core LSTM has the same kind of constraint (multiples of 64, CudaCaller.h:60-63)
        throw std::invalid_argument(large() ? "batch_size must be a multiple of 32 for this LSTM size"
                                              : "batch_size must be a multiple of 16 for LSTM models");
    }
    auto plan = std::make_unique<LstmPlan>();
    plan->model = this;
    if (const char* dbg = std::getenv("B200_DEBUG_LSTM_LAYERS")) plan->debug_layers = std::atoi(dbg);
    uint8_t* base = static_cast<uint8_t*>(ws);
    auto take = [&](size_t bytes) {
        uint8_t* p = base;
        base += (bytes + 255) & ~size_t(255);
        if ((size_t)(base - static_cast<uint8_t*>(ws)) > ws_bytes) throw std::logic_error("LSTM workspace overflow");
        return p;
    };
    const int Tp = t_pad(T_in);
    __half* x2 = reinterpret_cast<__half*>(take((size_t)N * Tp * 16 * 2));
    __half* seq = reinterpret_cast<__half*>(take((size_t)(T_out + 1) * Np * C * 2));
    __half* mid = desc.out_features > 0 ? reinterpret_cast<__half*>(take((size_t)T_out * Np * desc.out_features * 2)) : nullptr;
    __half* gxbuf = reinterpret_cast<__half*>(take((size_t)T_out * Np * 4 * C * 2));
    int* tile_counter = reinterpret_cast<int*>(take(256));

    // conv1 + conv2
    plan->conv12 = Conv12Params{signal, x2, conv_w, N, T_in, Tp, pad3(), desc.convs[0].size, desc.convs[0].winlen,
                                desc.convs[1].winlen, desc.convs[0].activation, desc.convs[1].activation, nullptr, tile_counter};
    plan->conv12_grid = dim3((T_in + CONV_TT - 1) / CONV_TT, N, 1);
    // the v5 shape runs conv2 on the tensor cores (conv12_tc_kernel); anything else keeps the FMA-pipe kernel
    // (B200_CONV12_FMA=1 forces it: the tests compare the two)
    plan->conv12_tc = desc.convs[0].size == 16 && desc.convs[1].winlen == 5 && !std::getenv("B200_CONV12_FMA");
    plan->conv12_tiles_per_chunk = (T_in + C12_TILE - 1) / C12_TILE;
    {
        const long long tiles = (long long)plan->conv12_tiles_per_chunk * N;
        plan->conv12_tc_grid = (int)std::min<long long>(tiles, 5LL * kNumSMs);
        if (plan->conv12_tc) ensure_dynamic_smem(conv12_tc_kernel, C12_SMEM);
    }

    // conv3: rows (n, t) read K3p contiguous halfs starting at x2[n][stride * t]
    {
        if (T_in % desc.stride != 0) throw std::invalid_argument("chunk size must be a multiple of the model stride");
        GemmDesc g{};
        g.a = x2;
        g.batches = N;
        g.rows_per_batch = T_out;
        g.a_row_stride = (int64_t)desc.convs[2].stride * 16;
        g.a_batch_stride = (int64_t)Tp * 16;
        g.w = w3;
        g.N = C;
        g.K = K3p;
        g.bias = b3;
        g.act = desc.convs[2].activation;
        g.out = seq;
        g.out_m1 = T_out;        // g = n * T_out + t
        g.out_s0 = C;            // n
        g.out_s1 = (int64_t)Np * C;  // t
        plan->conv3 = make_gemm_plan(g);
    }
    // LSTM layers: x-projection GEMM + cluster recurrence
    {
        plan->num_layers = desc.lstm_layers;
        plan->variable = variable_chunk_sizes();
        const int CL = rec_cluster(C);
        // Chunks per cluster: 32 for large batches, 16 below.  64 chunks (B200_CLUSTER_CHUNKS=64) spill registers next to
        // the register-resident W_hh of lstm_size 384 and were no faster: hac batch 512, 4 runners, 77.6 vs 77.7 Msamples/s
        // for 64 vs 32 (two alternating runs each, NVIDIA H100 80GB HBM3 at 700 W).  lstm_size 96 (one CTA per cluster)
        // stays at 16.
        int un = 16;
        if (CL > 1 && Np > 256) un = 32;
        if (const char* e = std::getenv("B200_CLUSTER_CHUNKS")) {   // tuning / A-B override
            const int v = std::atoi(e);
            if ((v == 16 || v == 32 || v == 64) && Np % v == 0) un = v;
            else throw std::invalid_argument("B200_CLUSTER_CHUNKS must be 16, 32 or 64 and divide the padded batch");
        }
        // one CTA of 8 x 96 threads cannot hold the accumulators of 64 chunks without spilling
        if (CL == 1 && un > 32) un = 32;
        while (Np % un != 0) un /= 2;
        plan->rec_un = un;
        plan->rec_ctas = (Np / un) * CL;
        // With three or more batches in flight the x-projection GEMMs keep off some SMs, so that another batch's recurrence
        // (several milliseconds of latency chain) can start beside them instead of queueing behind a GEMM that owns every SM.
        const int hint = num_runners_hint < 1 ? 1 : num_runners_hint;
        const int gemm_cap = hint >= 3 ? kNumSMs - 32 : 0;
        const int Cp = (C + 63) / 64 * 64;
        for (int l = 0; l < desc.lstm_layers; ++l) {
            GemmDesc g{};
            g.a = seq;   // rows (t, chunk), K = the layer input
            g.batches = 1;
            g.rows_per_batch = T_out * Np;
            g.a_row_stride = C;
            g.a_batch_stride = (int64_t)T_out * Np * C;
            g.a_inner = C;
            g.w = layers[l].w_ih;
            g.N = 4 * C;
            g.K = Cp;
            g.bias = layers[l].bias;
            g.act = GEMM_ACT_NONE;
            g.out = gxbuf;
            g.out_m1 = 1;
            g.out_s0 = 4 * C;
            g.max_ctas = gemm_cap;
            plan->gx_gemm.push_back(make_gemm_plan(g));
            LstmRecParams rp{};
            rp.seq = seq;
            rp.gx = gxbuf;
            rp.w_hh = layers[l].w_hh;
            rp.T = T_out;
            rp.N = Np;
            rp.reverse = (l % 2 == 0) ? 1 : 0;  // reverse_first = true (CRFModel.cpp:40, LSTMStack.cpp:31-41)
            rp.lens = nullptr;
            rp.stride = desc.stride;
            plan->rec_p.push_back(rp);
        }
    }
    // linear CRF (+ optional decomposition); rows g = t * Np + n  ->  scores[n][t][:]
    {
        GemmDesc g{};
        g.a = seq;
        g.batches = 1;
        g.rows_per_batch = T_out * Np;
        g.a_row_stride = C;
        g.a_batch_stride = (int64_t)T_out * Np * C;
        g.w = wl1;
        g.N = out1;
        g.K = Cp;
        g.a_inner = C;
        g.bias = bl1;
        if (desc.out_features > 0) {
            g.act = GEMM_ACT_NONE;
            g.out = mid;
            g.out_m1 = 1;
            g.out_s0 = out1;
            g.out_s1 = 0;
            plan->linear1 = make_gemm_plan(g);
            GemmDesc g2{};
            g2.a = mid;
            g2.batches = 1;
            g2.rows_per_batch = T_out * Np;
            g2.a_row_stride = out1;
            g2.a_batch_stride = (int64_t)T_out * Np * out1;
            g2.w = wl2;
            g2.N = desc.outsize;
            g2.K = out1;
            g2.act = desc.crf_scale == 5.0f ? GEMM_ACT_TANH_X5 : GEMM_ACT_NONE;
            g2.out = scores;
            g2.out_m1 = Np;
            g2.out_s0 = desc.outsize;
            g2.out_s1 = (int64_t)T_out * desc.outsize;
            plan->linear2 = make_gemm_plan(g2);
            plan->num_linear = 2;
        } else {
            g.act = desc.crf_scale == 5.0f ? GEMM_ACT_TANH_X5 : GEMM_ACT_NONE;
            g.out = scores;
            g.out_m1 = Np;                                  // g = t * Np + n
            g.out_s0 = desc.outsize;                        // t
            g.out_s1 = (int64_t)T_out * desc.outsize;       // n
            plan->linear1 = make_gemm_plan(g);
            plan->num_linear = 1;
        }
    }
    return plan;
}

template <int C, int CL, int NB>
static void launch_rec_t(const LstmRecParams& rp, int ctas, cudaStream_t stream) {
    using Cfg = RecCfg<C, CL, NB>;
    ensure_dynamic_smem(lstm_rec_kernel<C, CL, NB>, (int)Cfg::SMEM);
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)ctas, 1, 1);
    cfg.blockDim = dim3(Cfg::THREADS, 1, 1);
    cfg.dynamicSmemBytes = Cfg::SMEM;
    cfg.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = CL;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    B200_CUDA(cudaLaunchKernelEx(&cfg, lstm_rec_kernel<C, CL, NB>, rp));
}

template <int C>
static void launch_rec_c(const LstmRecParams& rp, int un, int ctas, cudaStream_t stream) {
    constexpr int CL = rec_cluster(C);
    switch (un) {
        case 64:
            if constexpr (CL > 1) launch_rec_t<C, CL, 64>(rp, ctas, stream);
            else throw std::logic_error("lstm recurrence: 64 chunks per single-CTA cluster");
            break;
        case 32: launch_rec_t<C, CL, 32>(rp, ctas, stream); break;
        default: launch_rec_t<C, CL, 16>(rp, ctas, stream); break;
    }
}

void LstmPlan::launch_rec(int l, cudaStream_t stream) const {
    switch (model->desc.lstm_size) {
        case 96: launch_rec_c<96>(rec_p[l], rec_un, rec_ctas, stream); break;
        case 192: launch_rec_c<192>(rec_p[l], rec_un, rec_ctas, stream); break;
        case 384: launch_rec_c<384>(rec_p[l], rec_un, rec_ctas, stream); break;
        default: throw Unsupported("no LSTM recurrence instantiation for this lstm_size");
    }
}

void LstmPlan::run(cudaStream_t stream, ProfileSink* prof) {
    {
        NvtxRange r("conv");
        if (conv12_tc) {
            B200_CUDA(cudaMemsetAsync(conv12.tile_counter, 0, sizeof(int), stream));
            conv12_tc_kernel<<<conv12_tc_grid, C12_THREADS, C12_SMEM, stream>>>(conv12, conv12_tiles_per_chunk,
                                                                                 conv12_tiles_per_chunk * conv12.N);
        } else {
            conv12_kernel<<<conv12_grid, CONV_TT, 0, stream>>>(conv12);
        }
        if (prof) prof->mark("conv12", stream);
        run_gemm(conv3, stream);
        if (prof) prof->mark("conv3_gemm", stream);
    }
    {
        NvtxRange lstm_range("lstm_stack");
        const int nl = debug_layers >= 0 && debug_layers < num_layers ? debug_layers : num_layers;
        for (int l = 0; l < nl; ++l) {
            NvtxRange r("lstm_layer");
            run_gemm(gx_gemm[l], stream);
            if (prof) prof->mark("lstm_gx_gemm", stream);
            launch_rec(l, stream);
            if (prof) prof->mark("lstm_rec", stream);
        }
        if (nl < num_layers) {  // debug: stop after nl layers (tools/debug_forward.py reads the sequence buffer)
            B200_CUDA(cudaGetLastError());
            return;
        }
    }
    NvtxRange r("linear");
    run_gemm(linear1, stream);
    if (prof) prof->mark("linear_gemm", stream);
    if (num_linear == 2) {
        run_gemm(linear2, stream);
        if (prof) prof->mark("linear2_gemm", stream);
    }
    B200_CUDA(cudaGetLastError());
}

}  // namespace

std::unique_ptr<Model> make_lstm_model(const b200_model_desc& desc, const b200_tensor* tensors, int n) {
    return std::make_unique<LstmModel>(desc, tensors, n);
}

}  // namespace b200
