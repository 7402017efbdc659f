// wgmma GEMM with fused epilogue:  out[row(g)][n] = act( sum_k A[g][k] * W[n][k] + bias[n] ), fp32 accumulation in
// registers (exact s32 for int8 operands).  GemmDesc::in_type and out_type name the element types; gemm.cu's table of kernel
// forms lists the combinations that run.
#pragma once

#include "tc.cuh"

namespace b200 {

enum GemmAct : int {
    GEMM_ACT_NONE = -1,
    GEMM_ACT_SWISH = 0,        // config::Activation::SWISH
    GEMM_ACT_SWISH_CLAMP = 1,  // SWISH_CLAMP (3.5)
    GEMM_ACT_TANH = 2,         // TANH
    GEMM_ACT_TANH_X5 = 3,      // tanh(x) * 5 (pre-v4.x CRF linear, dorado/nn/CRFModules.cpp:27-31)
    GEMM_ACT_SWIGLU = 4,       // columns (2j, 2j+1) = (y, gate) -> silu(gate) * y, N/2 outputs (TxModules.cpp:170-176)
    GEMM_ACT_ROPE = 5,         // output columns are [3][H][64] (q|k|v): rotary embedding on q and k (TxModules.cpp:220-250)
};

// Element type of the GEMM's operands (A and W) or of its output
enum GemmType : int {
    GEMM_F16 = 0,
    GEMM_E4M3 = 1,
    GEMM_S8 = 2,
};
// int8 value of an activation v in [-1, 1] (the last convolution's tanh output and every h_t of an int8 LSTM layer).  The
// reference's factor is inside closed Koi; 127 is this engine's choice: the symmetric range, so -128 never appears.
constexpr float kInt8ActScale = 127.0f;

struct GemmDesc {
    // in_type: A and W.  E4M3 and int8 take one byte per element, so a K block (one 128-byte TMA box row) is 128 elements
    // instead of 64 and K must be a multiple of 128.  int8 operands accumulate exactly in s32 and need col_scale [N], the
    // fp32 dequantisation factor per output column: v = float(acc) * col_scale[n] + bias[n].  With row_scale
    // [batches * rows_per_batch], the fp32 factor per A row, they take their own kernel forms:
    // v = (float(acc) * row_scale[g]) * col_scale[n] (+ bias[n]), each product rounded in fp32.
    // out_type: the stored element; out's strides count elements of it.  E4M3 goes with E4M3 operands and SwiGLU; int8 with
    // fp16 operands and tanh, stored as cvt.rni.sat(kInt8ActScale * tanh(v)).
    // gemm.cu's table lists the (in_type, out_type, act, row_scale set) forms and the optional inputs each one reads;
    // make_gemm_plan refuses any other combination, and any optional input the form does not read.
    GemmType in_type = GEMM_F16;
    GemmType out_type = GEMM_F16;
    const float* col_scale = nullptr;
    const float* row_scale = nullptr;
    // A: logical [batches][rows_per_batch][K] of in_type, K contiguous; row/batch strides in elements
    const void* a = nullptr;
    int batches = 1;
    int rows_per_batch = 0;
    int64_t a_row_stride = 0;
    int64_t a_batch_stride = 0;
    // W: [N][K] of in_type (K contiguous, row stride = K_pad)
    const void* w = nullptr;
    int N = 0;
    int K = 0;  // multiple of 64 (128 for E4M3 and int8; pad weights with zeros)
    int a_inner = 0;  // extent of A's K dimension in the tensor map (0 = K); elements beyond read as zero
    const float* bias = nullptr;
    int act = GEMM_ACT_NONE;
    // output: global row g = batch * rows_per_batch + row  ->  out + (g / out_m1) * out_s0 + (g % out_m1) * out_s1
    void* out = nullptr;   // out_type
    int64_t out_m1 = 1;
    int64_t out_s0 = 0;
    int64_t out_s1 = 0;
    // GEMM_ACT_ROPE: (cos, sin) table [T_max][32][2], tokens per chunk, number of leading columns to rotate
    const float* rope = nullptr;
    int rope_T = 0;
    int rope_cols = 0;
    int max_ctas = 0;      // > 0: persistent grid of at most this many CTAs (leave SMs to other runners' latency-bound kernels)
    int rope_stride = 0;   // positions per table row: the table is [16 dim pairs][rope_stride positions] float4 (cos, sin, cos, sin)
    // optional fused residual epilogue (deepnorm): v = v + alpha * residual[g][n]; requires act == NONE
    const __half* residual = nullptr;
    float alpha = 0.0f;
    // RMSNorm folded into the GEMMs around it (no separate pass, TxModules.cpp:667,712 koi_rmsnorm_residual):
    //   out_ss     the epilogue also writes, per output row, the sum of squares of the fp16 values it stored -- one partial
    //              per (column tile, epilogue part), summed in a fixed order by the consumers (deterministic, no atomics);
    //              out_ss_parts() gives how many partials a row has
    //   a_ss       A holds UN-normalised rows u: the accumulator row is scaled by rsqrt(mean(u^2) + eps) (the gain is folded
    //              into W's columns by the caller)
    //   res_ss/res_gain  the residual term is alpha * rsqrt(mean(u^2) + eps) * gain[n] * u[g][n]
    float* out_ss = nullptr;
    const float* a_ss = nullptr;
    int a_ss_parts = 0;
    const float* res_ss = nullptr;
    int res_ss_parts = 0;
    const float* res_gain = nullptr;
    int norm_dim = 0;
    float norm_eps = 1e-5f;
};

struct GemmPlan {
    CUtensorMap tma_a, tma_w;
    GemmDesc d;
    const void* kernel = nullptr;   // the descriptor's gemm_wgmma_kernel form
    int num_k_blocks = 0;
    int bn = 128;
    int tiles_per_batch = 0;
    dim3 grid;
    size_t smem = 0;
};

GemmPlan make_gemm_plan(const GemmDesc& d);
int gemm_out_ss_parts(int N);  // partial sums of squares per row a GEMM with N output columns writes (GemmDesc::out_ss)
void run_gemm(const GemmPlan& p, cudaStream_t stream);

}  // namespace b200
