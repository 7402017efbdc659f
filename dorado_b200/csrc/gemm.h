// wgmma GEMM with fused epilogue:  out[row(g)][n] = act( sum_k A[g][k] * W[n][k] + bias[n] ), fp16 in/out,
// fp32 accumulation in registers.  See gemm.cu.
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

struct GemmDesc {
    // A: logical [batches][rows_per_batch][K] fp16, K contiguous; row/batch strides in elements
    const __half* a = nullptr;
    int batches = 1;
    int rows_per_batch = 0;
    int64_t a_row_stride = 0;
    int64_t a_batch_stride = 0;
    // W: [N][K] fp16 (K contiguous, row stride = K_pad)
    const __half* w = nullptr;
    int N = 0;
    int K = 0;  // multiple of 64 (pad weights with zeros)
    int a_inner = 0;  // extent of A's K dimension in the tensor map (0 = K); elements beyond read as zero
    const float* bias = nullptr;
    int act = GEMM_ACT_NONE;
    // output: global row g = batch * rows_per_batch + row  ->  out + (g / out_m1) * out_s0 + (g % out_m1) * out_s1
    __half* out = nullptr;
    int64_t out_m1 = 1;
    int64_t out_s0 = 0;
    int64_t out_s1 = 0;
    // optional column blocking of the output: column n -> (n / out_col_m1) * out_col_s0 + (n % out_col_m1)
    // (out_col_m1 = 0: plain contiguous columns).  out_col_m1 must be a multiple of 32.
    int64_t out_col_m1 = 0;
    int64_t out_col_s0 = 0;
    int bias_per_row = 0;  // bias indexed by the global row g instead of the column
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
