// wgmma GEMM with fused epilogue:  out[row(g)][n] = act( sum_k A[g][k] * W[n][k] + bias[n] ), fp16 in/out (or E4M3
// operands, GemmDesc::fp8), fp32 accumulation in registers; or int8 operands with exact s32 accumulation and a per-column
// dequantisation factor (GemmDesc::q8).  See gemm.cu.
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

// The int8 precision of the LSTM models (GemmDesc::q8)
enum GemmQ8 : int {
    GEMM_Q8_NONE = 0,
    GEMM_Q8_OPERANDS = 1,  // A and W are int8: exact s32 accumulation, out = act(float(acc) * col_scale[n] + bias[n]) as fp16
                           // (float(acc) * row_scale[g] first when GemmDesc::row_scale is set)
    GEMM_Q8_STORE = 2,     // fp16 operands, GEMM_ACT_TANH: the output is int8 cvt.rni.sat(kInt8ActScale * tanh(v))
};
// int8 value of an activation v in [-1, 1] (the last convolution's tanh output and every h_t of an int8 LSTM layer).  The
// reference's factor is inside closed Koi; 127 is this engine's choice: the symmetric range, so -128 never appears.
constexpr float kInt8ActScale = 127.0f;

struct GemmDesc {
    // fp8 = 1: A and W are E4M3 bytes (K a multiple of 128, one 128-byte TMA box row per K block), and the SwiGLU epilogue
    // writes E4M3; every other epilogue writes fp16.  Only GEMM_ACT_NONE and GEMM_ACT_SWIGLU have E4M3 forms.
    int fp8 = 0;
    // q8: GemmQ8.  GEMM_Q8_OPERANDS takes int8 bytes with the E4M3 form's addressing (K a multiple of 128), the plain and
    // TANH_X5 activations, a column bias and col_scale [N] (fp32 dequantisation factor per output column).
    // GEMM_Q8_STORE writes int8 where the fp16 form writes fp16: out is int8 and its strides count bytes.
    // row_scale [batches * rows_per_batch] (optional, GEMM_Q8_OPERANDS only): fp32 dequantisation factor per A row, applied
    // as v = (float(acc) * row_scale[g]) * col_scale[n], each product rounded in fp32.  With it the form also takes
    // GEMM_ACT_ROPE (no bias), whose rotation then runs on v (the int8_qkv_fp8_ffn transformer's QKV projection).
    int q8 = GEMM_Q8_NONE;
    const float* col_scale = nullptr;
    const float* row_scale = nullptr;
    // A: logical [batches][rows_per_batch][K] fp16, K contiguous; row/batch strides in elements
    const void* a = nullptr;
    int batches = 1;
    int rows_per_batch = 0;
    int64_t a_row_stride = 0;
    int64_t a_batch_stride = 0;
    // W: [N][K] fp16 (K contiguous, row stride = K_pad)
    const void* w = nullptr;
    int N = 0;
    int K = 0;  // multiple of 64 (128 for fp8; pad weights with zeros)
    int a_inner = 0;  // extent of A's K dimension in the tensor map (0 = K); elements beyond read as zero
    const float* bias = nullptr;
    int act = GEMM_ACT_NONE;
    // output: global row g = batch * rows_per_batch + row  ->  out + (g / out_m1) * out_s0 + (g % out_m1) * out_s1
    void* out = nullptr;   // fp16, or E4M3 bytes (fp8 SwiGLU)
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
    int bn = 128;
    int tiles_per_batch = 0;
    dim3 grid;
    size_t smem = 0;
};

GemmPlan make_gemm_plan(const GemmDesc& d);
int gemm_out_ss_parts(int N);  // partial sums of squares per row a GEMM with N output columns writes (GemmDesc::out_ss)
void run_gemm(const GemmPlan& p, cudaStream_t stream);

}  // namespace b200
