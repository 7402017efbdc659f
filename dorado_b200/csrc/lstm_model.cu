// Conv -> LSTM -> linear CRF forward (fast / hac models) for sm_90a.
//
// Replaces, for the CUDA path of dorado/basecall/model/CRFModel.cpp:69-115:
//   ConvStack layers 1,2   host_convolution_f16              dorado/nn/ConvStack.cpp:216-232  -> conv12_tc_kernel (conv2 on
//                                                                                         mma.sync; v5 shapes), conv12_kernel (FMA pipe)
//   ConvStack layer 3      host_linear "cutlass conv"        dorado/nn/ConvStack.cpp:236-275  -> gemm.cu
//   LSTMStack              host_cutlass_lstm/host_small_lstm dorado/nn/LSTMStack.cpp:127-238 -> lstm_layer_kernel (lstm_size
//                                                                                         96), gx GEMM + lstm_rec_kernel (128, 192,
//                                                                                         256, 384),
//                                                                                         gx GEMM + lstm_grid_rec_kernel (768, 1024)
//   LinearCRF              host_linear                       dorado/nn/CRFModules.cpp:49-122   -> gemm.cu
//   int8 (CUTLASS_TNC_I8)  the same call sites with KOI_I8   ConvStack.cpp:66-74, LSTMStack.cpp:127-211, CRFModules.cpp:103-117
//                                                                                      -> the int8 forms of gemm.cu +
//                                                                                         lstm_rec_kernel (256, 384; opt-in)
// Semantics are those of the CPU modules (ConvStack.cpp:146-163, LSTMStack.cpp:29-41, CRFModules.cpp:24-34).
//
// The LSTM layers run through LstmStack (declared in lstm_kernels.h), which owns the layer weights' device layout, the
// recurrences' launch shapes, their counters and error word; the modified-base model (modbase_model.cu) runs its layers
// through the same stack.
//
// Activation layouts in HBM (fp16):
//   signal  [N][T_in]
//   x2      [N][T_in + 2*pad3 + 8][16]      conv2 output, NTC, zero rows = conv3's padding (+ K padding)
//   seq     [T_out][N][C]                   time-major LSTM buffer, updated in place by every layer (int8 in the int8_lstm
//                                           precision: cvt.rni.sat.s8(kInt8ActScale * v) of conv3's tanh output and every h_t)
//   scores  [N][T_out][outsize]
#include "engine.h"
#include "gemm.h"
#include "lstm_kernels.h"
#include "nvtx.h"
#include "tc.cuh"

#include <algorithm>
#include <cmath>
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
constexpr int MAXW = kConv12MaxWin;

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

}  // namespace

// conv1: torch [c1][1][w] -> [c1][w]; conv2: torch [co][ci][k] -> [k][ci][co]
float* upload_conv12_weights(const b200_tensor& tw, const b200_tensor& tb, const b200_tensor& tw2, const b200_tensor& tb2,
                             const b200_conv_desc& c1, const b200_conv_desc& c2) {
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
    return upload_f32(pk);
}

void launch_conv12(const Conv12Params& p, cudaStream_t stream) {
    conv12_kernel<<<dim3((p.T + CONV_TT - 1) / CONV_TT, p.N, 1), CONV_TT, 0, stream>>>(p);
}

namespace {

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

// Cell update of lstm_rec_kernel and lstm_grid_rec_kernel from the pre-activations i, f, g, o: updates the cell state c and
// returns h, both masked by alive (1, or 0 outside the chunk).  lstm_layer_kernel keeps a form of its own (fmaf, no mask).
__device__ __forceinline__ float lstm_cell(const float (&pre)[4], float& c, float alive) {
    const float ig = gate_act(pre[0], 1.0f), fg = gate_act(pre[1], 1.0f);
    const float gg = gate_act(pre[2], 2.0f), og = gate_act(pre[3], 1.0f);
    const float cs = (fg * c + ig * gg) * alive;
    c = cs;
    return og * tanh_f(cs) * alive;
}

// ------------------------------------------------------------------------------------------------
// lstm_size 96: one LSTM layer in one kernel (lstm_layer_kernel).
//
// A CTA of 12 warps owns 16 chunks for the whole sequence.  Warp w owns hidden units 8 w .. 8 w + 7 and all four of their
// gates: the host permutes the gate rows of W_ih, W_hh and the bias (lstm_fused_row) so that the warp's two m16 tiles are
// {i, f} and {g, o} of those 8 units.  An m16n8k16 accumulator then gives thread `lane` rows lane / 4 and lane / 4 + 8 of
// each tile, i.e. i, f, g and o of unit 8 w + lane / 4, for chunks 2 (lane % 4) (+ 1, + 8, + 9): the gate math runs from
// registers.  Both weight matrices stay in registers as A fragments (2 tiles x 6 K steps x 4 = 48 registers each).
//
// x_t is read in place from the sequence buffer (3 KB of 16 contiguous chunk rows per step), prefetched FL_AHEAD steps
// ahead into a shared-memory ring by cp.async.
//
// The 16 chunks are 16 independent recurrences, and the two n tiles have accumulators of their own: group A (n tile 0,
// chunks 0-7) and group B (n tile 1, chunks 8-15).  The groups run half a step apart, so that the tensor cores work on one
// group while the SFU runs the gate math of the other (one step with a single phase order leaves the tensor pipe idle
// during the gate math and the SFU idle during the MMAs).  Loop step s is
//     W_hh h_B(s-1)        ldmatrix of the B rows of h_s -> 12 mma.sync into ah_B, first read after barrier A
//     gates of A, step s   ah_A + gx_A -> cell update, h_A(s) -> h_s and the sequence buffer.  gx_A is W_ih x_A(s) + bias,
//                          rounded to fp16 as the x-projection GEMM of the larger sizes rounds gx
//     W_ih x_A(s+1)        ldmatrix of the A rows of the ring -> 12 mma.sync into ax_A, once the gates of A have read it
//     barrier A            publishes h_A(s)
//     W_hh h_A(s)          12 mma.sync into ah_A: the chain of A for step s + 1, first read after barrier B
//     gates of B, step s;  W_ih x_B(s+1)
//     prefetch x_{s+FL_AHEAD}; barrier B, which publishes h_B(s) and the ring slot of step s + 2
// The loop has no branch: the products of step T are computed in the last step and never read.  Nothing inside an
// accumulator changes order (k steps ascending), so the results do not depend on the schedule.
//
// Invariants:
// - h is ONE tile: the rows of A and B, each group with a single buffer.  Every read of h_X(s-1) and the write of h_X(s)
//   that overwrites it lie on the two sides of the other group's barrier: W_hh h_B(s-1) is read before barrier A of step
//   s and h_B(s) is written after it; W_hh h_A(s) is read after barrier A of step s and before barrier B of step s, and
//   h_A(s+1) is written after that.  The group's own barrier orders the write of h_X(s) before its read.  The prologue
//   reads h_A(-1) and ends with a CTA barrier of its own, before step 0 writes h_A(0).
// - ring: the cp.async of loop step s writes the slot of step s - 1.  Both groups read x(s-1) in loop step s - 2, before
//   its barrier B; the copy is issued after barrier B of step s - 1.
// - cp.async: before barrier B of loop step s every thread has waited for its copies of steps <= s + 2 (FL_AHEAD - 2
//   groups may stay in flight), and barrier B makes them visible.  Both groups read x(s+2) in loop step s + 1.
// - Writing h_t over x_t in the sequence buffer: both groups write h of step s in loop step s.  The copy of x(s) into the
//   ring completed before barrier B of loop step s - 2, and nothing reads x(s) from the sequence buffer after it.
// ------------------------------------------------------------------------------------------------
constexpr int FL_C = 96;
constexpr int FL_NB = 16;                   // chunks per CTA
constexpr int FL_THREADS = 32 * FL_C / 8;   // one warp per 8 hidden units
constexpr int FL_KS = FL_C / 16;            // K steps
constexpr int FL_HS = FL_C + 8;             // row stride (fp16) of h and x tiles: the 8 rows of an ldmatrix phase on distinct banks
constexpr int FL_TILE = FL_NB * FL_HS;      // one [chunk][unit] tile
constexpr int FL_GROUP_BYTES = 8 * FL_HS * 2;   // offset of the rows of group B in a tile
constexpr int FL_RING = 8;                  // x_t slots
// Steps between the cp.async of x_t and its use.  Step s copies into the slot of step s - 1.  The copy has to be complete
// at the end of step s + FL_AHEAD - 2, so it has FL_AHEAD - 2 steps to land.
constexpr int FL_AHEAD = FL_RING - 1;
constexpr int FL_X_COPIES = FL_NB * FL_C * 2 / 16;   // 16-byte copies per step

// permuted gate row of PyTorch row gate * C + unit (gate order i | f | g | o): warp unit / 8, tile gate / 2, half gate % 2
__host__ __device__ constexpr int lstm_fused_row(int gate, int unit) { return (unit / 8) * 32 + gate * 8 + unit % 8; }

struct LstmLayerParams {
    __half* seq;          // [T][N][C] layer input, overwritten with h in place
    const __half* w_ih;   // [4C][C], rows permuted (lstm_fused_row)
    const __half* w_hh;   // [4C][C], rows permuted
    const float* bias;    // [4C] b_ih + b_hh, permuted
    int T, N, reverse;
};

__global__ void __launch_bounds__(FL_THREADS, 1) lstm_layer_kernel(const LstmLayerParams p) {
    constexpr int C = FL_C, NB = FL_NB, KS = FL_KS, HS = FL_HS;
    __shared__ __align__(16) __half h_s[FL_TILE];            // h of both groups
    __shared__ __align__(16) __half x_s[FL_RING * FL_TILE];  // x_t ring
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n0 = blockIdx.x * NB;
    const int T = p.T;

    // x of step s -> ring slot s % FL_RING; threads 0 .. FL_X_COPIES - 1 copy 16 bytes each.  Every thread commits one
    // group per step (empty if it copies nothing), so that the group counts of cp_async_wait agree across threads.
    auto prefetch_x = [&](int s) {
        if (s < T && threadIdx.x < FL_X_COPIES) {
            const int t = p.reverse ? T - 1 - s : s;
            const int n = threadIdx.x / (C / 8), col = threadIdx.x % (C / 8) * 8;
            tc::cp_async_16(tc::smem_u32(x_s + (s % FL_RING) * FL_TILE + n * HS + col),
                            p.seq + ((size_t)t * p.N + n0 + n) * C + col);
        }
        tc::cp_async_commit();
    };
    for (int s = 0; s < FL_AHEAD; ++s) prefetch_x(s);
    for (int i = threadIdx.x; i < FL_TILE / 8; i += FL_THREADS) reinterpret_cast<uint4*>(h_s)[i] = make_uint4(0, 0, 0, 0);

    // A fragments of tile mt (gates 2 mt, 2 mt + 1): rows warp * 32 + mt * 16 + lane / 4 (+ 8)
    uint32_t wh[2][KS][4], wi[2][KS][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
        const int r_lo = warp * 32 + mt * 16 + (lane >> 2), r_hi = r_lo + 8;
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
            const int col = ks * 16 + 2 * (lane & 3);
            const int off[4] = {r_lo * C + col, r_hi * C + col, r_lo * C + col + 8, r_hi * C + col + 8};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                wh[mt][ks][j] = __ldg(reinterpret_cast<const unsigned int*>(p.w_hh + off[j]));
                wi[mt][ks][j] = __ldg(reinterpret_cast<const unsigned int*>(p.w_ih + off[j]));
            }
        }
    }
    const int unit = warp * 8 + (lane >> 2);
    float bias[4];
#pragma unroll
    for (int g = 0; g < 4; ++g) bias[g] = __ldg(p.bias + lstm_fused_row(g, unit));
    float c_reg[2][2] = {{0.0f, 0.0f}, {0.0f, 0.0f}};  // [group][chunk of the pair]

    // ldmatrix.x4 over two k steps of one group's 8 rows: matrix qm = (k step qm / 2, k half qm % 2), row qr
    const int qm = lane >> 3, qr = lane & 7;
    const uint32_t frag_off = (uint32_t)((qr * HS + qm * 8) * 2);
    const uint32_t h_frag = tc::smem_u32(h_s) + frag_off, x_frag = tc::smem_u32(x_s) + frag_off;
    // acc[mt] = A[mt] x (the 8 chunk rows at `rows`), K = C in ascending k steps: n tile `group` of the gate layout above
    auto mma_group = [&](float (*acc)[4], const uint32_t (*a)[KS][4], uint32_t rows) {
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) acc[mt][0] = acc[mt][1] = acc[mt][2] = acc[mt][3] = 0.0f;
#pragma unroll
        for (int kp = 0; kp < KS / 2; ++kp) {
            uint32_t b[4];
            tc::ldmatrix_x4(b, rows + kp * 64);
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) tc::mma_f16_16816(acc[mt], a[mt][2 * kp], b[0], b[1]);
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) tc::mma_f16_16816(acc[mt], a[mt][2 * kp + 1], b[2], b[3]);
        }
    };
    float ah[2][2][4], ax[2][2][4];  // [group][tile][element]: W_hh h and W_ih x of the group's next gates

    // Gates of group g at one step: gate `gate` of the cell (g, e) is tile gate / 2, row half gate % 2 -> accumulator
    // element 2 (gate % 2) + e.  ax[g] is read first and then refilled with W_ih x of the next step from ring slot x_next.
    auto gates = [&](const int g, __half* out, const uint32_t x_next) {
        float pre[2][4];
#pragma unroll
        for (int gate = 0; gate < 4; ++gate) {
            const int mt = gate >> 1, j = 2 * (gate & 1);
            const float2 gx = __half22float2(__floats2half2_rn(ax[g][mt][j] + bias[gate], ax[g][mt][j + 1] + bias[gate]));
            pre[0][gate] = ah[g][mt][j] + gx.x;
            pre[1][gate] = ah[g][mt][j + 1] + gx.y;
        }
        mma_group(ax[g], wi, x_next + g * FL_GROUP_BYTES);
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const float ig = gate_act(pre[e][0], 1.0f), fg = gate_act(pre[e][1], 1.0f);
            const float gg = gate_act(pre[e][2], 2.0f), og = gate_act(pre[e][3], 1.0f);
            const float cs = fmaf(ig, gg, fg * c_reg[g][e]);  // fused explicitly, so that its rounding is fixed
            c_reg[g][e] = cs;
            const __half hv = __float2half_rn(og * tanh_f(cs));
            const int n = g * 8 + 2 * (lane & 3) + e;
            h_s[n * HS + unit] = hv;
            out[(size_t)n * C] = hv;
        }
    };
    tc::cp_async_wait<FL_AHEAD - 2>();  // x of steps 0 and 1
    __syncthreads();
    mma_group(ax[0], wi, x_frag);
    mma_group(ax[1], wi, x_frag + FL_GROUP_BYTES);
    mma_group(ah[0], wh, h_frag);  // h_A(-1) = 0
    __syncthreads();               // every warp has read h_A(-1) before step 0 writes h_A(0) over it

    for (int s = 0; s < T; ++s) {
        const int t = p.reverse ? T - 1 - s : s;
        __half* out = p.seq + ((size_t)t * p.N + n0) * C + unit;
        const uint32_t x_next = x_frag + ((s + 1) % FL_RING) * FL_TILE * 2;
        mma_group(ah[1], wh, h_frag + FL_GROUP_BYTES);
        gates(0, out, x_next);
        named_bar_sync(1, FL_THREADS);  // barrier A
        mma_group(ah[0], wh, h_frag);
        gates(1, out, x_next);
        prefetch_x(s + FL_AHEAD);
        tc::cp_async_wait<FL_AHEAD - 2>();  // x of step s + 2 has landed (this thread's part)
        named_bar_sync(2, FL_THREADS);  // barrier B
    }
}

// ------------------------------------------------------------------------------------------------
// LSTM layer = hoisted x-projection + recurrence (lstm_size 128, 192, 256 and 384).
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
// C = 128 and 192 split over clusters of 4 CTAs, 256 and 384 over clusters of 8 (32 or 48 hidden units per CTA, 256 or 384
// threads).
//
// The int8 form (I8; lstm_size 256 and 384, the int8_lstm precision) runs the same steps on int8 operands:
//   * W_hh rows are int8 (quantised per gate row, quantize_rows_f16) and stay in registers as mma.sync m16n8k32 A fragments:
//     C / 32 x 4 registers per thread, half of the fp16 form's;
//   * h is int8 in shared memory and in the sequence buffer.  An ldmatrix 8x8 b16 tile reads 16 bytes of K from each of 8
//     chunk rows, which is the s8 B fragment;
//   * the s32 accumulator is exact.  The MMA warp converts it and multiplies by inv[row] = 1 / (kInt8ActScale * scale[row])
//     (fp32), so the gate buffer holds fp32 W_hh h_{t-1} as in the fp16 form, and pre = that + gx;
//   * h_t is quantised once, cvt.rni.sat.s8(kInt8ActScale * h): the same byte pair goes to every CTA's copy of h and to the
//     sequence buffer.
// Counted in bytes the two forms address memory alike: a K step is 32 bytes of a W_hh row and of an h row (k16 fp16, k32
// int8), and a row of h is C elements at a stride of C elements + 16 bytes, 16 (mod 128), which puts the 8 rows of an
// ldmatrix phase on distinct banks.
// ------------------------------------------------------------------------------------------------

// CTAs per cluster for a hidden size: the CTA's W_hh rows (4 C / CL x C fp16) must fit its registers
__host__ __device__ constexpr int rec_cluster(int C) { return C <= 192 ? 4 : 8; }

// Parameters of lstm_rec_kernel and lstm_grid_rec_kernel
struct LstmRecParams {
    void* seq;              // [T][N][C] output h (in place over the layer input, which gx has consumed): fp16, int8 in the int8 form
    const __half* gx;       // [T][N][4C]
    const void* w_hh;       // [4C][C], PyTorch row order: fp16, int8 in the int8 form
    int T, N, reverse;
    const int32_t* lens;    // optional per-chunk length in samples (variable chunk sizes); stride = samples per step
    int stride;
    // lstm_grid_rec_kernel only
    int n_first;            // first chunk of this launch; group g owns chunks n_first + g NB ..
    unsigned int* counters; // one arrival counter per group of this launch, zero at launch
    int* error;             // set to 1 when a group barrier times out
    // the int8 form of lstm_rec_kernel only
    const float* inv;       // [4C] dequantisation factor of a gate row's accumulator
};

template <bool I8, int C, int CL, int NB>
struct RecCfg {
    using T = std::conditional_t<I8, int8_t, __half>;   // element of W_hh and h
    static constexpr int EB = (int)sizeof(T);     // bytes per element
    static constexpr int U = C / CL;              // hidden units per CTA
    static constexpr int MT = 4 * U / 16;         // m16 tiles of gate rows = warps
    static constexpr int THREADS = 32 * MT;
    static constexpr int KE = 32 / EB;            // K of one MMA: 32 bytes (k16 fp16, k32 int8)
    static constexpr int KS = C / KE;             // K steps
    static constexpr int NT = NB / 8;             // n8 tiles of chunks
    static constexpr int HS = C + 16 / EB;        // row stride of h in elements: the 8 rows of an ldmatrix phase on distinct banks
    static constexpr int GS = NB + 4;             // row stride of the gate pre-activations (fp32)
    static constexpr int PAIRS = U / 2 * NB / THREADS;   // (unit pair, chunk) cells per thread
    // gx is loaded ahead of the MMAs when it fits the registers; with 4 cell pairs per thread (64 chunks per cluster) the
    // 16 extra registers would spill, so gx is loaded in the cell loop instead
    static constexpr bool GX_AHEAD = PAIRS <= 2;
    static constexpr size_t SMEM = (size_t)2 * NB * HS * EB + (size_t)4 * U * GS * 4;
    static_assert(C % KE == 0 && C % CL == 0 && U % 4 == 0 && NT % 2 == 0 && PAIRS >= 1 && (U / 2 * NB) % THREADS == 0,
                  "recurrence shape");
    static_assert(HS * EB % 128 == 16 && THREADS <= 1024 && CL > 1 && CL <= 8, "h stride / block / cluster size");
};

template <bool I8, int C, int CL, int NB>
__global__ void __launch_bounds__(RecCfg<I8, C, CL, NB>::THREADS, 1) lstm_rec_kernel(const LstmRecParams p) {
    using Cfg = RecCfg<I8, C, CL, NB>;
    using T = typename Cfg::T;
    using Acc = std::conditional_t<I8, int32_t, float>;     // MMA accumulator
    using H2 = std::conditional_t<I8, uint16_t, __half2>;   // h of a unit pair
    constexpr int U = Cfg::U, EB = Cfg::EB, KE = Cfg::KE, KS = Cfg::KS, NT = Cfg::NT, HS = Cfg::HS, GS = Cfg::GS;
    constexpr int PAIRS = Cfg::PAIRS;
    constexpr bool GX_AHEAD = Cfg::GX_AHEAD;
    extern __shared__ __align__(16) uint8_t smem_raw[];
    T* h_s = reinterpret_cast<T*>(smem_raw);                                      // [2][NB][HS]  this CTA's copy of h
    float* g_s = reinterpret_cast<float*>(smem_raw + (size_t)2 * NB * HS * EB);   // [4U][GS]
    T* seq = static_cast<T*>(p.seq);
    __shared__ int len_s[NB];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    cg::cluster_group cluster = cg::this_cluster();
    const int rank = (int)cluster.block_rank();
    const int n0 = (int)(blockIdx.x / CL) * NB;
    if (threadIdx.x < NB) len_s[threadIdx.x] = p.lens ? min(p.T, __ldg(p.lens + n0 + threadIdx.x) / p.stride) : p.T;
    for (int i = threadIdx.x; i < 2 * NB * HS * EB / 16; i += Cfg::THREADS) reinterpret_cast<uint4*>(h_s)[i] = make_uint4(0, 0, 0, 0);

    // A fragments: local gate row r <-> W_hh row (r / U) * C + rank * U + r % U; in the int8 form also inv[] of rows r_lo, r_hi
    uint32_t a[KS][4];
    float inv_lo = 0.0f, inv_hi = 0.0f;
    {
        const int r_lo = warp * 16 + (lane >> 2), r_hi = r_lo + 8;
        const int g_lo = (r_lo / U) * C + rank * U + r_lo % U, g_hi = (r_hi / U) * C + rank * U + r_hi % U;
        const T* w_lo = static_cast<const T*>(p.w_hh) + (size_t)g_lo * C;
        const T* w_hi = static_cast<const T*>(p.w_hh) + (size_t)g_hi * C;
        if constexpr (I8) {
            inv_lo = __ldg(p.inv + g_lo);
            inv_hi = __ldg(p.inv + g_hi);
        }
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
            const int col = ks * KE + 4 / EB * (lane & 3);
            a[ks][0] = __ldg(reinterpret_cast<const unsigned int*>(w_lo + col));
            a[ks][1] = __ldg(reinterpret_cast<const unsigned int*>(w_hi + col));
            a[ks][2] = __ldg(reinterpret_cast<const unsigned int*>(w_lo + col + KE / 2));
            a[ks][3] = __ldg(reinterpret_cast<const unsigned int*>(w_hi + col + KE / 2));
        }
    }
    // accumulator -> fp32 W_hh h_{t-1} of the gate buffer (the int8 form dequantises its exact s32 sum per gate row)
    auto gate_sum = [](Acc v, float inv) -> float {
        if constexpr (I8) return (float)v * inv;
        else return v;
    };
    // cells: pair index q = threadIdx.x + j * THREADS -> units (u, u + 1), u = 2 (q % (U / 2)), chunk q / (U / 2)
    float c_reg[PAIRS][2];
#pragma unroll
    for (int j = 0; j < PAIRS; ++j) c_reg[j][0] = c_reg[j][1] = 0.0f;
    // every CTA of the cluster has zeroed its copy of h before anybody writes h_0 into it
    cluster.sync();

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
        Acc acc[NT][4];
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0;
        const uint32_t hb = tc::smem_u32(h_s + cur * NB * HS);
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
#pragma unroll
            for (int np = 0; np < NT / 2; ++np) {
                uint32_t b[4];
                const int n = (2 * np + (qm >> 1)) * 8 + qr, k = ks * KE + (qm & 1) * (KE / 2);
                tc::ldmatrix_x4(b, hb + (uint32_t)((n * HS + k) * EB));
                if constexpr (I8) {
                    tc::mma_s8_16832(acc[2 * np], a[ks], b[0], b[1]);
                    tc::mma_s8_16832(acc[2 * np + 1], a[ks], b[2], b[3]);
                } else {
                    tc::mma_f16_16816(acc[2 * np], a[ks], b[0], b[1]);
                    tc::mma_f16_16816(acc[2 * np + 1], a[ks], b[2], b[3]);
                }
            }
        }
        {
            const int r_lo = warp * 16 + (lane >> 2);
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) {
                const int col = nt * 8 + 2 * (lane & 3);
                *reinterpret_cast<float2*>(g_s + r_lo * GS + col) =
                        make_float2(gate_sum(acc[nt][0], inv_lo), gate_sum(acc[nt][1], inv_lo));
                *reinterpret_cast<float2*>(g_s + (r_lo + 8) * GS + col) =
                        make_float2(gate_sum(acc[nt][2], inv_hi), gate_sum(acc[nt][3], inv_hi));
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
            // h_t of the unit pair: fp32, or quantised as cvt.rni.sat.s8(kInt8ActScale * h) in the int8 form
            std::conditional_t<I8, int32_t, float> hv[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                float pre[4];
#pragma unroll
                for (int g = 0; g < 4; ++g) {
                    const float2 x = __half22float2(gxj[g]);
                    pre[g] = g_s[(g * U + u + e) * GS + n] + (e ? x.y : x.x);
                }
                const float h = lstm_cell(pre, c_reg[j][e], alive);
                if constexpr (I8) hv[e] = tc::cvt_rni_sat_s8(kInt8ActScale * h);
                else hv[e] = h;
            }
            H2 h2;
            if constexpr (I8) h2 = (uint16_t)((hv[0] & 0xff) | ((hv[1] & 0xff) << 8));
            else h2 = __floats2half2_rn(hv[0], hv[1]);
            *reinterpret_cast<H2*>(seq + ((size_t)t * p.N + n0 + n) * C + rank * U + u) = h2;
            T* h_own = h_s + (nxt * NB + n) * HS + rank * U + u;
#pragma unroll
            for (int r = 0; r < CL; ++r) *reinterpret_cast<H2*>(cluster.map_shared_rank(h_own, r)) = h2;
        }
        // h_t has landed in every copy, and every thread is done with h_{t-1} and the gate buffer
        cluster.sync();
    }
}

// ------------------------------------------------------------------------------------------------
// lstm_size 768 and 1024: recurrence over a group of CTAs that exchange h through L2 (lstm_grid_rec_kernel).
//
// W_hh is 4.5 MiB (768) or 8 MiB (1024) of fp16, more than the registers and shared memory of a cluster, so the weights are
// spread over a group of G = C / 16 CTAs, one per SM: CTA `rank` owns hidden units [16 rank, 16 rank + 16), i.e. the 64
// gate rows i, f, g, o of those units (64 x C fp16 = 96 or 128 KiB), in registers for the whole sequence.  Warp w holds
// the m16 tile of gate w % 4 over K half w / 4 (C / 32 k steps x 4 registers per thread); the two K halves are summed in
// shared memory.  A group owns NB chunks.  A step is
//     gx of this thread's cells -> registers    (independent of the recurrence: in flight during the wait)
//     wait until all G CTAs of the group have arrived after the previous step (counter >= G s)
//     h_{t-1} of the NB chunks: cp.async.cg (L2, not L1) from the sequence buffer, where the group wrote it
//     G[64][NB] = W_hh[rows of this CTA] h_{t-1}    mma.sync m16n8k16, B fragments by ldmatrix
//     gates, cell update (fp32 cell state in registers), h_t (fp16) -> the sequence buffer
//     arrive: CTA barrier, then one thread: fence + red.release.gpu add 1 on the group's counter
// h_t goes in place over the layer input x_t, which the x-projection GEMM has consumed; each step writes a new row of the
// sequence buffer, so one barrier per step orders everything.  The counter wait is bounded: a CTA that waits longer
// than GR_SPIN_BUDGET cycles, or finds the error word set, sets the error word and returns (the host turns it into an
// error).  The host launches a grid of whole groups that can all be resident at once (cooperative launch).
// ------------------------------------------------------------------------------------------------
constexpr int GR_UNITS = 16;     // hidden units per CTA
constexpr int GR_THREADS = 256;  // 8 warps: gate = warp % 4, K half = warp / 4
constexpr long long GR_SPIN_BUDGET = 2000000000LL;  // clock64 cycles: about one second at the H100's 1.98 GHz

template <int C, int NB>
struct GridCfg {
    static constexpr int G = C / GR_UNITS;                 // CTAs per group
    static constexpr int KS = C / 2 / 16;                  // k steps per warp (one K half)
    static constexpr int NT = NB / 8;                      // n8 tiles of chunks
    static constexpr int HS = C + 8;                       // row stride of h (fp16): an ldmatrix phase on distinct banks
    static constexpr int GS = NB + 4;                      // row stride of the partial gate sums (fp32)
    static constexpr int PAIRS = GR_UNITS / 2 * NB / GR_THREADS;  // (unit pair, chunk) cells per thread
    static constexpr size_t SMEM = (size_t)NB * HS * 2 + (size_t)2 * 4 * GR_UNITS * GS * 4;
    static_assert(C % (2 * 16) == 0 && NT % 2 == 0 && PAIRS >= 1 && (GR_UNITS / 2 * NB) % GR_THREADS == 0, "grid shape");
};

template <int C, int NB>
__global__ void __launch_bounds__(GR_THREADS, 1) lstm_grid_rec_kernel(const LstmRecParams p) {
    using Cfg = GridCfg<C, NB>;
    constexpr int G = Cfg::G, KS = Cfg::KS, NT = Cfg::NT, HS = Cfg::HS, GS = Cfg::GS, PAIRS = Cfg::PAIRS;
    constexpr int U = GR_UNITS;
    extern __shared__ __align__(16) uint8_t smem_raw[];
    __half* h_s = reinterpret_cast<__half*>(smem_raw);                             // [NB][HS]  h_{t-1}
    float* g_s = reinterpret_cast<float*>(smem_raw + (size_t)NB * HS * 2);         // [K half][4U gate rows][GS]
    __half* seq = static_cast<__half*>(p.seq);
    __shared__ int len_s[NB];
    __shared__ int abort_s;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int gate = warp & 3, kh = warp >> 2;
    const int group = (int)blockIdx.x / G, rank = (int)blockIdx.x % G;
    const int n0 = p.n_first + group * NB;
    unsigned int* counter = p.counters + group;
    if (threadIdx.x < NB) len_s[threadIdx.x] = p.lens ? min(p.T, __ldg(p.lens + n0 + threadIdx.x) / p.stride) : p.T;

    // A fragments: W_hh rows gate * C + U rank + lane / 4 (+ 8), columns of K half kh
    uint32_t a[KS][4];
    {
        const __half* w_lo = static_cast<const __half*>(p.w_hh) + (size_t)(gate * C + rank * U + (lane >> 2)) * C + kh * (C / 2);
        const __half* w_hi = w_lo + (size_t)8 * C;
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
            const int col = ks * 16 + 2 * (lane & 3);
            a[ks][0] = __ldg(reinterpret_cast<const unsigned int*>(w_lo + col));
            a[ks][1] = __ldg(reinterpret_cast<const unsigned int*>(w_hi + col));
            a[ks][2] = __ldg(reinterpret_cast<const unsigned int*>(w_lo + col + 8));
            a[ks][3] = __ldg(reinterpret_cast<const unsigned int*>(w_hi + col + 8));
        }
    }
    // cells: pair index q = threadIdx.x + j * GR_THREADS -> units (u, u + 1), u = 2 (q % (U / 2)), chunk q / (U / 2)
    float c_reg[PAIRS][2];
#pragma unroll
    for (int j = 0; j < PAIRS; ++j) c_reg[j][0] = c_reg[j][1] = 0.0f;
    __syncthreads();
    int steps = 0;
    for (int i = 0; i < NB; ++i) steps = max(steps, len_s[i]);
    const int qm = lane >> 3, qr = lane & 7;   // ldmatrix: matrix qm = (n tile qm / 2, k half qm % 2), row qr

    for (int s = 0; s < steps; ++s) {
        const int t = p.reverse ? steps - 1 - s : s;
        __half2 gxv[PAIRS][4];
#pragma unroll
        for (int j = 0; j < PAIRS; ++j) {
            const int q = threadIdx.x + j * GR_THREADS;
            const int u = 2 * (q % (U / 2)), n = q / (U / 2);
            const __half* gp = p.gx + ((size_t)t * p.N + n0 + n) * (4 * C) + rank * U + u;
#pragma unroll
            for (int g = 0; g < 4; ++g) gxv[j][g] = *reinterpret_cast<const __half2*>(gp + g * C);
        }
        if (s == 0) {
            for (int i = threadIdx.x; i < NB * HS / 8; i += GR_THREADS) reinterpret_cast<uint4*>(h_s)[i] = make_uint4(0, 0, 0, 0);
        } else {
            // every CTA of the group has stored h_{t-1} (step s - 1)
            if (threadIdx.x == 0) {
                const unsigned int target = (unsigned int)(G * s);
                const long long start = clock64();
                int failed = 0;
                while (tc::ld_acquire_gpu(counter) < target) {
                    if (tc::ld_relaxed_gpu(p.error) != 0 || clock64() - start > GR_SPIN_BUDGET) {
                        failed = 1;
                        break;
                    }
                }
                if (failed) atomicExch(p.error, 1);
                abort_s = failed;
            }
            __syncthreads();
            if (abort_s) return;
            const int tp = p.reverse ? t + 1 : t - 1;
            const __half* src = seq + ((size_t)tp * p.N + n0) * C;
            for (int i = threadIdx.x; i < NB * C / 8; i += GR_THREADS) {
                const int n = i / (C / 8), col = i % (C / 8) * 8;
                tc::cp_async_16(tc::smem_u32(h_s + n * HS + col), src + (size_t)n * C + col);
            }
            tc::cp_async_commit();
            tc::cp_async_wait<0>();
        }
        __syncthreads();
        float acc[NT][4];
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.0f;
        const uint32_t hb = tc::smem_u32(h_s) + (uint32_t)(kh * (C / 2) * 2);
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
            float* gw = g_s + (kh * 4 * U + gate * U + (lane >> 2)) * GS;
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) {
                const int col = nt * 8 + 2 * (lane & 3);
                *reinterpret_cast<float2*>(gw + col) = make_float2(acc[nt][0], acc[nt][1]);
                *reinterpret_cast<float2*>(gw + 8 * GS + col) = make_float2(acc[nt][2], acc[nt][3]);
            }
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < PAIRS; ++j) {
            const int q = threadIdx.x + j * GR_THREADS;
            const int u = 2 * (q % (U / 2)), n = q / (U / 2);
            // outside the chunk (variable chunk sizes) the state is held at zero: a multiplicative mask, not a branch
            const float alive = t < len_s[n] ? 1.0f : 0.0f;
            float hv[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                float pre[4];
#pragma unroll
                for (int g = 0; g < 4; ++g) {
                    const float2 x = __half22float2(gxv[j][g]);
                    const int row = (g * U + u + e) * GS + n;
                    pre[g] = (g_s[row] + g_s[4 * U * GS + row]) + (e ? x.y : x.x);
                }
                hv[e] = lstm_cell(pre, c_reg[j][e], alive);
            }
            *reinterpret_cast<__half2*>(seq + ((size_t)t * p.N + n0 + n) * C + rank * U + u) = __floats2half2_rn(hv[0], hv[1]);
        }
        // arrive: the CTA's h_t stores precede the release; the barrier also ends every read of h_s and g_s of this step
        __syncthreads();
        if (threadIdx.x == 0) {
            __threadfence();
            tc::red_release_gpu_add(counter, 1u);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// host side: the LSTM stack
// ------------------------------------------------------------------------------------------------
// A launch of `ctas` CTAs with one launch attribute, `at` (a cluster dimension or the cooperative flag)
static cudaLaunchConfig_t launch_config(int ctas, int threads, size_t smem, cudaStream_t stream, cudaLaunchAttribute& at) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)ctas, 1, 1);
    cfg.blockDim = dim3((unsigned)threads, 1, 1);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cfg.attrs = &at;
    cfg.numAttrs = 1;
    return cfg;
}

template <bool I8, int C, int NB>
static void launch_rec_t(const LstmRecParams& p, int ctas, cudaStream_t stream) {
    constexpr int CL = rec_cluster(C);
    using Cfg = RecCfg<I8, C, CL, NB>;
    ensure_dynamic_smem(lstm_rec_kernel<I8, C, CL, NB>, (int)Cfg::SMEM);
    cudaLaunchAttribute at{};
    at.id = cudaLaunchAttributeClusterDimension;
    at.val.clusterDim = {CL, 1, 1};
    const cudaLaunchConfig_t cfg = launch_config(ctas, Cfg::THREADS, Cfg::SMEM, stream, at);
    B200_CUDA(cudaLaunchKernelEx(&cfg, lstm_rec_kernel<I8, C, CL, NB>, p));
}

// Launches lstm_rec_kernel<int8, C, cluster, nb> over `ctas` CTAs; throws Unsupported for a shape without an instantiation
void launch_lstm_rec(bool int8, int C, int nb, int ctas, const LstmRecParams& p, cudaStream_t stream) {
    static constexpr struct {
        bool int8;
        int C, nb;
        void (*launch)(const LstmRecParams&, int, cudaStream_t);
    } kRec[] = {
        {false, 128, 16, launch_rec_t<false, 128, 16>},
        {false, 128, 32, launch_rec_t<false, 128, 32>},
        {false, 128, 64, launch_rec_t<false, 128, 64>},
        {false, 192, 16, launch_rec_t<false, 192, 16>},
        {false, 192, 32, launch_rec_t<false, 192, 32>},
        {false, 192, 64, launch_rec_t<false, 192, 64>},
        {false, 256, 16, launch_rec_t<false, 256, 16>},
        {false, 256, 32, launch_rec_t<false, 256, 32>},
        {false, 256, 64, launch_rec_t<false, 256, 64>},
        {false, 384, 16, launch_rec_t<false, 384, 16>},
        {false, 384, 32, launch_rec_t<false, 384, 32>},
        {false, 384, 64, launch_rec_t<false, 384, 64>},
        {true, 256, 16, launch_rec_t<true, 256, 16>},
        {true, 256, 32, launch_rec_t<true, 256, 32>},
        {true, 256, 64, launch_rec_t<true, 256, 64>},
        {true, 384, 16, launch_rec_t<true, 384, 16>},
        {true, 384, 32, launch_rec_t<true, 384, 32>},
        {true, 384, 64, launch_rec_t<true, 384, 64>},
    };
    for (const auto& k : kRec) {
        if (k.int8 == int8 && k.C == C && k.nb == nb) return k.launch(p, ctas, stream);
    }
    throw Unsupported(std::string("no ") + (int8 ? "int8 " : "") + "LSTM recurrence instantiation for this lstm_size");
}

// Chunks per cluster: 32 for large batches, 16 below.  64 chunks (B200_CLUSTER_CHUNKS=64) spill registers next to the
// register-resident W_hh of lstm_size 384 and were no faster: hac batch 512, 4 runners, 77.6 vs 77.7 Msamples/s for 64 vs 32
// (two alternating runs each, NVIDIA H100 80GB HBM3 at 700 W).
int lstm_rec_chunks(int Np) {
    int un = Np > 256 ? 32 : 16;
    if (const char* e = std::getenv("B200_CLUSTER_CHUNKS")) {   // tuning / A-B override
        const int v = std::atoi(e);
        if ((v == 16 || v == 32 || v == 64) && Np % v == 0) un = v;
        else throw std::invalid_argument("B200_CLUSTER_CHUNKS must be 16, 32 or 64 and divide the padded batch");
    }
    while (Np % un != 0) un /= 2;
    return un;
}

// lstm_grid_rec_kernel<C, nb> and its dynamic shared memory (set as the kernel's limit)
struct GridKernel {
    const void* fn;
    size_t smem;
};
template <int C, int NB>
static GridKernel grid_kernel() {
    ensure_dynamic_smem(lstm_grid_rec_kernel<C, NB>, (int)GridCfg<C, NB>::SMEM);
    return {reinterpret_cast<const void*>(lstm_grid_rec_kernel<C, NB>), GridCfg<C, NB>::SMEM};
}
static GridKernel grid_kernel(int C, int nb) {
    switch (C * 100 + nb) {
        case 76832: return grid_kernel<768, 32>();
        case 76864: return grid_kernel<768, 64>();
        case 102432: return grid_kernel<1024, 32>();
        case 102464: return grid_kernel<1024, 64>();
        default: throw Unsupported("no grid LSTM recurrence instantiation for this lstm_size");
    }
}

// A cooperative launch: the driver refuses a grid whose CTAs cannot all be resident at once instead of starting part of it
void launch_lstm_grid(int C, int nb, int ctas, const LstmRecParams& p, cudaStream_t stream) {
    const GridKernel k = grid_kernel(C, nb);
    cudaLaunchAttribute at{};
    at.id = cudaLaunchAttributeCooperative;
    at.val.cooperative = 1;
    const cudaLaunchConfig_t cfg = launch_config(ctas, GR_THREADS, k.smem, stream, at);
    void* args[] = {const_cast<LstmRecParams*>(&p)};
    B200_CUDA(cudaLaunchKernelExC(&cfg, k.fn, args));
}

// Groups of lstm_grid_rec_kernel that fit the GPU at once: every CTA of a launch must be resident, because CTAs wait for
// each other at every step.
static int grid_max_groups(int C, int nb) {
    int dev = 0, sms = 0, per_sm = 0;
    B200_CUDA(cudaGetDevice(&dev));
    B200_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const GridKernel k = grid_kernel(C, nb);
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k.fn, GR_THREADS, k.smem));
    return per_sm * sms / (C / GR_UNITS);
}

// Launch shape of lstm_grid_rec_kernel for a padded batch of Np chunks (a multiple of 32), when max_groups groups fit the
// GPU at once: NB chunks per group, groups per launch, launches per layer (each launch a whole recurrence over its chunks).
// nb > 0 and groups > 0 replace the choice of NB and of the groups per launch (B200_GRID_CHUNKS, B200_GRID_GROUPS).
struct GridShape {
    int nb, groups, launches;
};
GridShape grid_shape(int Np, int max_groups32, int max_groups64, int runners, int nb, int groups) {
    // 64 chunks per group when that still fills every resident group: half the barriers per chunk
    if (nb <= 0) nb = (max_groups64 >= 1 && Np % 64 == 0 && Np / 64 >= max_groups64) ? 64 : 32;
    const int max_groups = nb == 64 ? max_groups64 : max_groups32;
    const int tiles = Np / nb;
    // with R batches in flight, each batch's recurrence takes ~1/R of the SMs and runs beside the others' kernels
    groups = std::min(tiles, groups > 0 ? groups : std::max(1, max_groups / std::max(1, runners)));
    return {nb, groups, (tiles + groups - 1) / groups};
}

}  // namespace

// fp32 PyTorch layouts -> LstmLayerWeights: gate rows permuted by lstm_fused_row for lstm_size 96, W_ih's K padded to a
// multiple of 64 for the x-projection GEMM of the other sizes
LstmLayerWeights upload_lstm_layer(int C, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh) {
    const bool fused = C == FL_C;
    const int Kp = fused ? C : (C + 63) / 64 * 64;
    std::vector<float> wi((size_t)4 * C * Kp, 0.0f), wh((size_t)4 * C * C), b((size_t)4 * C);
    for (int r = 0; r < 4 * C; ++r) {
        const int dst = fused ? lstm_fused_row(r / C, r % C) : r;
        std::memcpy(&wi[(size_t)dst * Kp], &w_ih[(size_t)r * C], sizeof(float) * C);
        std::memcpy(&wh[(size_t)dst * C], &w_hh[(size_t)r * C], sizeof(float) * C);
        b[dst] = b_ih[r] + b_hh[r];
    }
    LstmLayerWeights w;
    w.w_ih = upload_f16(wi);
    w.w_hh = upload_f16(wh);
    w.bias = upload_f32(b);
    return w;
}

// utils::quantize_tensor(w, 1) (torch_utils/tensor_utils.cpp:293-300) as torch evaluates it on an fp16 tensor: every
// operation computes in fp32 and rounds its result to fp16.  128 / absmax, the product w * scale and its rounding to the
// nearest integer (ties to even) are all fp16 values.  An all-zero row gives the reference 128 / 0 = inf and NaN products;
// here such a row gets q = 0, and its callers give it a dequantisation factor of 0.
static float f16_to_float(uint16_t bits) {
    __half_raw r;
    r.x = bits;
    return __half2float(__half(r));
}
void quantize_rows_f16(const uint16_t* w16, int rows, int cols, int8_t* q, uint16_t* scale16) {
    for (int r = 0; r < rows; ++r) {
        const uint16_t* w = w16 + (size_t)r * cols;
        float absmax = 0.0f;
        for (int c = 0; c < cols; ++c) absmax = std::max(absmax, std::fabs(f16_to_float(w[c])));
        scale16[r] = f16_bits(128.0f / absmax);   // +inf for an all-zero row
        const float scale = f16_to_float(scale16[r]);
        for (int c = 0; c < cols; ++c) {
            if (absmax == 0.0f) {
                q[(size_t)r * cols + c] = 0;
                continue;
            }
            const float prod = f16_to_float(f16_bits(f16_to_float(w[c]) * scale));
            q[(size_t)r * cols + c] = (int8_t)std::min(127.0f, std::max(-127.0f, std::nearbyintf(prod)));
        }
    }
}
// Factor that turns an s32 accumulator of int8 activations (kInt8ActScale * v) and a row's int8 weights back into W v
float int8_row_inv(uint16_t scale16) {
    const float s = f16_to_float(scale16);
    return std::isinf(s) ? 0.0f : 1.0f / (kInt8ActScale * s);
}

template <typename T>
static T* upload_raw(const std::vector<T>& v) {
    T* d = nullptr;
    B200_CUDA(cudaMalloc(&d, v.size() * sizeof(T)));
    B200_CUDA(cudaMemcpy(d, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
    return d;
}

// The int8 form (lstm_size 256 and 384): fp16(W_ih) | fp16(W_hh) quantised as one [4C][2C] matrix, one scale per gate row
// of both (LSTMStack.cpp:150-166)
LstmLayerWeights upload_lstm_layer_int8(int C, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh) {
    const int R = 4 * C;
    std::vector<uint16_t> both((size_t)R * 2 * C), scale(R);
    for (int r = 0; r < R; ++r) {
        for (int c = 0; c < C; ++c) {
            both[(size_t)r * 2 * C + c] = f16_bits(w_ih[(size_t)r * C + c]);
            both[(size_t)r * 2 * C + C + c] = f16_bits(w_hh[(size_t)r * C + c]);
        }
    }
    std::vector<int8_t> q((size_t)R * 2 * C), qi((size_t)R * C), qh((size_t)R * C);
    quantize_rows_f16(both.data(), R, 2 * C, q.data(), scale.data());
    std::vector<float> inv(R), b(R);
    for (int r = 0; r < R; ++r) {
        std::memcpy(&qi[(size_t)r * C], &q[(size_t)r * 2 * C], C);
        std::memcpy(&qh[(size_t)r * C], &q[(size_t)r * 2 * C + C], C);
        inv[r] = int8_row_inv(scale[r]);
        b[r] = b_ih[r] + b_hh[r];
    }
    LstmLayerWeights w;
    w.w_ih8 = upload_raw(qi);
    w.w_hh8 = upload_raw(qh);
    w.inv = upload_f32(inv);
    w.bias = upload_f32(b);
    return w;
}

void free_lstm_layer(LstmLayerWeights& w) {
    cudaFree(w.w_ih);
    cudaFree(w.w_hh);
    cudaFree(w.bias);
    cudaFree(w.w_ih8);
    cudaFree(w.w_hh8);
    cudaFree(w.inv);
    w = LstmLayerWeights{};
}

LstmStackBuffers carve_lstm_stack(Bump& b, int C, int num_layers, int T, int Np) {
    LstmStackBuffers w;
    if (C == FL_C) return w;  // the fused layer computes gx in registers
    w.gx = b.take<__half>((size_t)T * Np * 4 * C * 2);
    if (C > 384) {  // lstm_grid_rec_kernel: at most one arrival counter per 32 chunks and layer, and the error word
        w.counter_bytes = (size_t)num_layers * (Np / 32) * sizeof(unsigned int);
        w.counters = b.take<unsigned int>(w.counter_bytes);
        w.error = b.take<int>(sizeof(int));
    }
    return w;
}

LstmStack::LstmStack(const LstmStackDesc& d, const LstmStackBuffers& ws) : m_d(d), m_ws(ws) {
    const int C = d.C, Np = d.Np;
    if (d.int8 && C != 256 && C != 384) throw Unsupported("the int8 LSTM layers exist for lstm_size 256 and 384 only");
    if (const char* dbg = std::getenv("B200_DEBUG_LSTM_LAYERS")) m_debug_layers = std::atoi(dbg);
    if (C == FL_C) {  // one lstm_layer_kernel per layer
        m_nb = FL_NB;
        m_groups = Np / FL_NB;
        return;
    }
    if (C <= 384) {  // one cluster per m_nb chunks, all in one launch
        m_kind = Kind::Rec;
        m_nb = lstm_rec_chunks(Np);
        m_groups = Np / m_nb;
        m_group_ctas = rec_cluster(C);
    } else {
        // B200_GRID_CHUNKS (32 or 64) and B200_GRID_GROUPS override the shape, for tuning and for the tests that compare shapes
        m_kind = Kind::Grid;
        const int mg32 = grid_max_groups(C, 32), mg64 = grid_max_groups(C, 64);
        if (mg32 < 1) throw Unsupported("lstm_size " + std::to_string(C) + ": one group of CTAs does not fit this GPU");
        const char* env_nb = std::getenv("B200_GRID_CHUNKS");
        const char* env_groups = std::getenv("B200_GRID_GROUPS");
        const int nb = env_nb ? std::atoi(env_nb) : 0, groups = env_groups ? std::atoi(env_groups) : 0;
        if (env_nb && ((nb != 32 && nb != 64) || Np % nb != 0 || (nb == 64 && mg64 < 1))) {
            throw std::invalid_argument("B200_GRID_CHUNKS must be 32 or 64 and divide the padded batch");
        }
        const GridShape s = grid_shape(Np, mg32, mg64, d.runners, nb, groups);
        if (env_groups && (groups < 1 || groups > (s.nb == 64 ? mg64 : mg32))) {
            throw std::invalid_argument("B200_GRID_GROUPS must be 1 .. the resident groups");
        }
        m_nb = s.nb;
        m_groups = s.groups;
        m_launches = s.launches;
        m_group_ctas = C / GR_UNITS;
    }
    // With three or more batches in flight the x-projection GEMMs keep off some SMs, so that another batch's recurrence
    // (several milliseconds of latency chain) can start beside them instead of queueing behind a GEMM that owns every SM.
    const int gemm_cap = d.runners >= 3 ? kNumSMs - 32 : 0;
    for (int l = 0; l < d.num_layers; ++l) {
        const LstmLayerWeights& w = d.layers[l];
        GemmDesc g{};
        g.a = d.seq;   // rows (t, chunk), K = the layer input
        g.batches = 1;
        g.rows_per_batch = d.T * Np;
        g.a_row_stride = C;
        g.a_batch_stride = (int64_t)d.T * Np * C;
        g.a_inner = C;
        g.w = w.w_ih;
        g.N = 4 * C;
        g.K = (C + 63) / 64 * 64;
        if (d.int8) {   // rows of int8, K = C = whole 128-byte blocks
            g.in_type = GEMM_S8;
            g.w = w.w_ih8;
            g.col_scale = w.inv;
            g.K = C;
        }
        g.bias = w.bias;
        g.act = GEMM_ACT_NONE;
        g.out = m_ws.gx;
        g.out_m1 = 1;
        g.out_s0 = 4 * C;
        g.max_ctas = gemm_cap;
        m_gx_gemm.push_back(make_gemm_plan(g));
    }
    if (m_ws.error) {
        B200_CUDA(cudaMemset(m_ws.error, 0, sizeof(int)));
        B200_CUDA(cudaHostAlloc(&m_error_host, sizeof(int), cudaHostAllocDefault));
        *m_error_host = 0;
    }
}

LstmStack::~LstmStack() {
    if (m_error_host) cudaFreeHost(m_error_host);
}

bool LstmStack::run(cudaStream_t stream, ProfileSink* prof) {
    NvtxRange stack_range("lstm_stack");
    auto mark = [&](const char* name) {
        if (prof) prof->mark(name, stream);
    };
    const int C = m_d.C, Np = m_d.Np;
    if (m_ws.counters) B200_CUDA(cudaMemsetAsync(m_ws.counters, 0, m_ws.counter_bytes, stream));
    const int nl = m_debug_layers >= 0 && m_debug_layers < m_d.num_layers ? m_debug_layers : m_d.num_layers;
    for (int l = 0; l < nl; ++l) {
        NvtxRange r("lstm_layer");
        const LstmLayerWeights& w = m_d.layers[l];
        const int reverse = (l % 2 == 0) == m_d.reverse_first ? 1 : 0;
        if (m_kind == Kind::Layer) {
            lstm_layer_kernel<<<m_groups, FL_THREADS, 0, stream>>>(
                    LstmLayerParams{static_cast<__half*>(m_d.seq), w.w_ih, w.w_hh, w.bias, m_d.T, Np, reverse});
            mark("lstm_layer");
            continue;
        }
        run_gemm(m_gx_gemm[l], stream);
        mark(m_d.int8 ? "lstm_gx_gemm_i8" : "lstm_gx_gemm");
        const void* w_hh = m_d.int8 ? static_cast<const void*>(w.w_hh8) : w.w_hh;
        // launch i covers groups i * m_groups .. of m_nb chunks, with counters of its own (the last may hold fewer groups)
        for (int i = 0; i < m_launches; ++i) {
            const int ctas = std::min(m_groups, Np / m_nb - i * m_groups) * m_group_ctas;
            unsigned int* counters = m_ws.counters ? m_ws.counters + (size_t)l * (Np / 32) + (size_t)i * m_groups : nullptr;
            const LstmRecParams p{m_d.seq, m_ws.gx, w_hh, m_d.T, Np, reverse, m_lens, m_d.stride, i * m_groups * m_nb,
                                  counters, m_ws.error, w.inv};
            if (m_kind == Kind::Rec) {
                launch_lstm_rec(m_d.int8, C, m_nb, ctas, p, stream);
                mark(m_d.int8 ? "lstm_rec_i8" : "lstm_rec");
            } else {
                launch_lstm_grid(C, m_nb, ctas, p, stream);
                mark("lstm_grid_rec");
            }
        }
    }
    // the error word of the grid recurrence, read by check_errors() once the stream has drained
    if (m_error_host) B200_CUDA(cudaMemcpyAsync(m_error_host, m_ws.error, sizeof(int), cudaMemcpyDeviceToHost, stream));
    return nl == m_d.num_layers;
}

void LstmStack::check_errors() {
    if (!m_error_host || *m_error_host == 0) return;
    *m_error_host = 0;
    B200_CUDA(cudaMemset(m_ws.error, 0, sizeof(int)));
    throw std::runtime_error("lstm_grid_rec_kernel: a group of CTAs did not reach its step barrier within the time "
                             "budget; the outputs of this batch are invalid");
}

std::string LstmStack::info() const {
    const std::string ctas = std::to_string(m_groups * m_group_ctas);
    switch (m_kind) {
        case Kind::Layer: return "lstm_layer.ctas=" + ctas;
        case Kind::Rec:
            return "lstm_rec.ctas=" + ctas + ";lstm_rec.chunks_per_cluster=" + std::to_string(m_nb) + (m_d.int8 ? ";lstm.int8=1" : "");
        default:
            return "lstm_grid.ctas=" + ctas + ";lstm_grid.groups=" + std::to_string(m_groups) + ";lstm_grid.chunks_per_group=" +
                   std::to_string(m_nb) + ";lstm_grid.launches_per_layer=" + std::to_string(m_launches);
    }
}

int LstmStack::launches() const { return m_d.num_layers * (m_kind == Kind::Layer ? 1 : 1 + m_launches); }

// ------------------------------------------------------------------------------------------------
// host side: the basecaller
// ------------------------------------------------------------------------------------------------
namespace {

class LstmPlan final : public ForwardPlan {
public:
    void run(cudaStream_t stream, ProfileSink* prof) override;
    int launches() const override { return 1 + 1 + lstm->launches() + num_linear; }
    std::string info() const override { return lstm->info(); }   // "lstm.int8=1" among them in the int8_lstm precision
    void set_chunk_lengths(const int32_t* d_lens) override {
        if (!variable) return;  // the mode exists for the models that run variable chunk sizes only
        conv12.lens = d_lens;
        lstm->set_chunk_lengths(d_lens);
    }
    void check_errors() override { lstm->check_errors(); }

    Conv12Params conv12{};
    dim3 conv12_grid;
    bool conv12_tc = false;  // conv2 on the tensor cores (conv12_tc_kernel)
    int conv12_tiles_per_chunk = 0, conv12_tc_grid = 0;
    GemmPlan conv3;
    bool variable = false;
    std::unique_ptr<LstmStack> lstm;
    GemmPlan linear1, linear2;
    int num_linear = 1;
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
    // desc.lstm_precision == B200_LSTM_INT8: int8 sequence buffer, int8 LSTM layers (layers[].w_ih8 ...), and the first
    // linear on int8 operands: wl1_8 [out1][C] quantised per output row, wl1_inv [out1] (wl1 unused)
    bool int8 = false;
    int8_t* wl1_8 = nullptr;
    float* wl1_inv = nullptr;

private:
    struct Buffers {
        __half* x2;    // conv2 output [N][t_pad][16]: first, the tests read it at offset 0
        void* seq;     // [T_out + 1][Np][C] fp16 (int8 in the int8_lstm precision): second, the tests read it right behind x2
        __half* mid;   // decomposition only: [T_out][Np][out_features]
        int* tile_counter;  // conv12_tc_kernel
        LstmStackBuffers lstm;
    };
    // The workspace layout for N chunks of T_in samples; refuses a batch the LSTM kernels cannot take
    Buffers carve(Bump& b, int N, int T_in) const;
    int pad3() const { return desc.convs[2].winlen / 2; }
    int t_pad(int T_in) const { return T_in + 2 * pad3() + 8; }
    // lstm_size 96 keeps the reference's fixed-size contract (batch a multiple of 16, no variable chunk sizes); the larger
    // sizes, 128 included, take batches in multiples of 32 and variable chunk sizes
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
    if (C != 96 && C != 128 && C != 192 && C != 256 && C != 384 && C != 768 && C != 1024) {
        // kernels are instantiated for the sizes of the reference's model zoo this engine covers
        throw Unsupported("lstm_size " + std::to_string(C) + " is not supported (96, 128, 192, 256, 384, 768 and 1024 are)");
    }

    if (d.lstm_layers < 1 || d.lstm_layers > 8) throw std::invalid_argument("bad lstm_layers");
    int8 = d.lstm_precision == B200_LSTM_INT8;
    if (int8) {
        // The reference's CUTLASS_TNC_I8 conditions (ConvStack.cpp:66-74) cut down to the int8 lstm_rec_kernel's widths
        if (C != 256 && C != 384) {
            throw Unsupported("int8_lstm precision: lstm_size " + std::to_string(C) + " is not supported (256 and 384 are)");
        }
        if (c3.activation != B200_ACT_TANH) {
            throw Unsupported("int8_lstm precision needs a tanh last convolution: the int8 activations assume values in [-1, 1]");
        }
        if (d.lstm_inner_dim > 0) throw Unsupported("int8_lstm precision: FLSTM models (lstm_inner_dim > 0) are not supported");
    }

    conv_w = upload_conv12_weights(find_tensor(tensors, n, "0.conv.weight.tensor"), find_tensor(tensors, n, "0.conv.bias.tensor"),
                                   find_tensor(tensors, n, "1.conv.weight.tensor"), find_tensor(tensors, n, "1.conv.bias.tensor"),
                                   c1, c2);
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
    // LSTM layers
    for (int l = 0; l < d.lstm_layers; ++l) {
        const std::string pfx = std::to_string(d.num_convs + l + 1) + ".rnn.";
        // plain LSTM: the tensors as they are.  FLSTM (nn/FLSTMStack.cpp:18-25,108-124): gates = up_ih (dn_ih x_t) +
        // up_hh (dn_hh h_{t-1}) + bias, folded once into W = up x dn (double accumulation, rounded to fp32) so that the
        // same LSTM kernels serve both model kinds.
        std::vector<float> folded_ih, folded_hh;
        const float *wih, *whh, *bih, *bhh;
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
            wih = folded_ih.data();
            whh = folded_hh.data();
            bih = find_tensor(tensors, n, pfx + "up_bias_ih.tensor").data;
            bhh = find_tensor(tensors, n, pfx + "up_bias_hh.tensor").data;
        } else {
            wih = find_tensor(tensors, n, pfx + "weight_ih_l0.tensor").data;
            whh = find_tensor(tensors, n, pfx + "weight_hh_l0.tensor").data;
            bih = find_tensor(tensors, n, pfx + "bias_ih_l0.tensor").data;
            bhh = find_tensor(tensors, n, pfx + "bias_hh_l0.tensor").data;
        }
        layers.push_back(int8 ? upload_lstm_layer_int8(C, wih, whh, bih, bhh) : upload_lstm_layer(C, wih, whh, bih, bhh));
    }
    // linear(s)
    {
        const int layer = d.num_convs + d.lstm_layers + 1;
        const auto& tw = find_tensor(tensors, n, std::to_string(layer) + ".linear.weight.tensor");
        out1 = d.out_features > 0 ? d.out_features : d.outsize;
        Cp = (C + 63) / 64 * 64;
        std::vector<float> w((size_t)out1 * Cp, 0.0f);
        for (int o = 0; o < out1; ++o) std::memcpy(&w[(size_t)o * Cp], &tw.data[(size_t)o * C], sizeof(float) * C);
        if (int8) {   // quantised per output row, as CRFModules.cpp:107-109 (C is a multiple of 128: no K padding)
            std::vector<uint16_t> w16((size_t)out1 * C), scale(out1);
            for (size_t i = 0; i < w16.size(); ++i) w16[i] = f16_bits(tw.data[i]);
            std::vector<int8_t> q(w16.size());
            quantize_rows_f16(w16.data(), out1, C, q.data(), scale.data());
            std::vector<float> inv(out1);
            for (int o = 0; o < out1; ++o) inv[o] = int8_row_inv(scale[o]);
            wl1_8 = upload_raw(q);
            wl1_inv = upload_f32(inv);
        } else {
            wl1 = upload_f16(w);
        }
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
    for (auto& l : layers) free_lstm_layer(l);
    cudaFree(wl1);
    cudaFree(wl1_8);
    cudaFree(wl1_inv);
    cudaFree(bl1);
    cudaFree(wl2);
}

LstmModel::Buffers LstmModel::carve(Bump& b, int N, int T_in) const {
    const int C = desc.lstm_size;
    const int T_out = T_in / desc.stride;
    const int Np = n_pad(N);
    if (Np != N) {
        // the reference's tensor-core LSTM has the same kind of constraint (multiples of 64, CudaCaller.h:60-63)
        throw std::invalid_argument(large() ? "batch_size must be a multiple of 32 for this LSTM size"
                                              : "batch_size must be a multiple of 16 for LSTM models");
    }
    Buffers w;
    w.x2 = b.take<__half>((size_t)N * t_pad(T_in) * 16 * 2);
    w.seq = b.take((size_t)(T_out + 1) * Np * C * (int8 ? 1 : 2));
    w.mid = desc.out_features > 0 ? b.take<__half>((size_t)T_out * Np * desc.out_features * 2) : nullptr;
    w.tile_counter = b.take<int>(sizeof(int));
    w.lstm = carve_lstm_stack(b, C, desc.lstm_layers, T_out, Np);
    return w;
}

size_t LstmModel::workspace_bytes(int N, int T_in) const {
    Bump sizing;
    carve(sizing, N, T_in);
    return sizing.used();
}

std::unique_ptr<ForwardPlan> LstmModel::make_plan(int N, int T_in, const __half* signal, __half* scores, void* ws,
                                                  size_t ws_bytes) {
    const int C = desc.lstm_size;
    const int T_out = T_in / desc.stride;
    const int Np = n_pad(N);
    Bump b(ws, ws_bytes);
    const auto [x2, seq, mid, tile_counter, lstm_ws] = carve(b, N, T_in);
    if (b.used() != ws_bytes) throw std::logic_error("LSTM workspace: the plan's layout differs from workspace_bytes()");
    auto plan = std::make_unique<LstmPlan>();
    const int Tp = t_pad(T_in);

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
        g.out_type = int8 ? GEMM_S8 : GEMM_F16;
        g.out = seq;
        g.out_m1 = T_out;        // g = n * T_out + t
        g.out_s0 = C;            // n
        g.out_s1 = (int64_t)Np * C;  // t
        plan->conv3 = make_gemm_plan(g);
    }
    plan->variable = variable_chunk_sizes();
    LstmStackDesc lstm{};
    lstm.C = C;
    lstm.T = T_out;
    lstm.Np = Np;
    lstm.stride = desc.stride;
    lstm.runners = num_runners_hint;
    lstm.reverse_first = true;  // CRFModel.cpp:40, LSTMStack.cpp:31-41
    lstm.int8 = int8;
    lstm.seq = seq;
    lstm.layers = layers.data();
    lstm.num_layers = desc.lstm_layers;
    plan->lstm = std::make_unique<LstmStack>(lstm, lstm_ws);
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
        if (int8) {
            g.in_type = GEMM_S8;
            g.w = wl1_8;
            g.col_scale = wl1_inv;
            g.K = C;
        }
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
    if (!lstm->run(stream, prof)) {  // debug: stopped after B200_DEBUG_LSTM_LAYERS layers (tools/debug_forward.py)
        B200_CUDA(cudaGetLastError());
        return;
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
