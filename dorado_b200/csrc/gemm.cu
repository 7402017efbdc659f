// wgmma GEMM for the dense layers of the basecaller (last conv as a strided GEMM, CRF linear, LSTM input projection and
// every transformer projection).  Successor of the reference's cuBLAS/Koi call sites:
//   matmul_f16 (cublasGemmEx)      dorado/torch_utils/cuda_utils.cpp:386-403
//   host_linear / cutlass conv     dorado/nn/ConvStack.cpp:257, dorado/nn/CRFModules.cpp:112
//   koi_linear / koi_mm_swiglu     dorado/nn/TxModules.cpp:653-697
//
// Persistent: one CTA per SM loops over 128 x BN output tiles (BN <= 128).  Warpgroup 0 is the TMA producer (one thread:
// A and W tiles, 128-byte swizzle, a STAGES-deep mbarrier ring that runs across tiles); warpgroups 1 and 2 own rows 0-63 and
// 64-127 of the tile: they issue wgmma m64n32k16 straight from the swizzled stages, keep the fp32 accumulator in registers
// and run the epilogue (bias / activation / residual / rotary / SwiGLU -> fp16 -> global) from the accumulator fragments.
// The kernel's template names its form: activation, operand type, output type and row factors (kForms below lists the 14
// forms that are built).  E4M3 operands (the transformer's fc1 / fc2 in the fp8_ffn precision): the same ring, tiles and
// epilogues with 128 E4M3 per 128-byte K row instead of 64 fp16, wgmma m64n32k32.e4m3 and the SwiGLU output cast to E4M3.
// int8 operands (the x-projection and the CRF linear of LSTM models in the int8_lstm precision): the E4M3 form's ring and
// boxes, wgmma m64n32k32.s8 into s32 accumulators, which the epilogue converts and multiplies by a per-column fp32 factor
// (and by a per-row one in the forms with row factors: the transformer's QKV + RoPE projection in the int8_qkv_fp8_ffn
// precision).  The int8 output goes with fp16 operands: the tanh epilogue stores int8 (those models' last conv).
// A is addressed through a 3-D tensor map (k, row, batch) so that overlapping-row views work: the last conv of the LSTM
// models reads its im2col rows straight from the NTC activation buffer with row stride = stride * C_in (the reference's
// "cutlass_conv" trick, ConvStack.cpp:236-275).
#include "gemm.h"

#include "common.cuh"
#include "engine.h"

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <string>
#include <type_traits>
#include <vector>

namespace b200 {

namespace {

constexpr int BM = 128;
constexpr int BK = 64;              // fp16 per K block: one 128-byte swizzle row
constexpr int BK8 = 128;            // E4M3 or int8 per K block
constexpr int BN_MAX = 128;
constexpr int STAGES = 5;          // TMA -> wgmma ring depth: 5 x 32 KB of the 227 KB
constexpr int GEMM_PARTS = 4;      // RMSNorm partial sums per row and column tile (GemmDesc::out_ss): one per 32-column chunk
constexpr int GEMM_THREADS = 384;  // warpgroup 0: producer; warpgroups 1, 2: MMA + epilogue of 64 rows each

struct GemmKernelParams {
    int rows_per_batch, tiles_per_batch, N, num_k_blocks, bn;
    int num_tiles, n_tiles, m_tiles;  // total tiles, tiles along N, row tiles (all batches)
    int mfast;                        // row tile index runs fastest (fewer row tiles than column tiles)
    const float* bias;
    __half* out;
    uint32_t out_m1;
    long long out_s0, out_s1;
    const float* rope;
    int rope_T, rope_cols, rope_stride;
    const __half* residual;
    float alpha;
    // RMSNorm folded into the epilogue (GemmDesc)
    float* out_ss;
    const float* a_ss;
    const float* res_ss;
    const float* res_gain;
    int a_ss_parts, res_ss_parts;
    float norm_inv_dim, norm_eps;
    const float* col_scale;   // int8 operands
    const float* row_scale;   // int8 operands, the forms with row factors
};

// i-th tile of this CTA: row tile mt, column tile nt; false when the CTA has run out of tiles.  Producer and consumers walk
// the same sequence.  CTAs take consecutive tiles, and the SHORTER dimension runs fastest, so that the CTAs working at any
// moment share their tiles of the long operand (read from HBM once, then served by L2) and sweep the long operand once.
__device__ __forceinline__ bool gemm_tile_at(const GemmKernelParams& p, int i, int* mt, int* nt) {
    const int tile = (int)blockIdx.x + i * (int)gridDim.x;
    if (p.mfast) {
        *mt = tile % p.m_tiles;
        *nt = tile / p.m_tiles;
    } else {
        *mt = tile / p.n_tiles;
        *nt = tile % p.n_tiles;
    }
    return tile < p.num_tiles;
}

// The activation is a template parameter of the kernel: with a run-time switch inside the unrolled epilogue loops the
// compiler if-converts it and every element pays for every variant's ex2 / rcp.
template <int ACT>
__device__ __forceinline__ float act_apply(float v) {
    if constexpr (ACT == GEMM_ACT_SWISH) return swish_fast(v);
    else if constexpr (ACT == GEMM_ACT_SWISH_CLAMP) return fminf(swish_fast(v), 3.5f);
    else if constexpr (ACT == GEMM_ACT_TANH) return tanh_fast(v);
    else if constexpr (ACT == GEMM_ACT_TANH_X5) return 5.0f * tanh_fast(v);
    else return v;
}

// One K block (128 bytes: 64 fp16 or 128 E4M3) of a warpgroup's 64 x 32 NCH tile: 32 rows of W are 4 KB further on,
// 32 bytes along K (16 fp16, 32 E4M3: one wgmma) are +2 in the (addr >> 4) field of a descriptor.
template <int NCH, bool FP8, typename Acc>
__device__ __forceinline__ void wgmma_k_block(Acc (&acc)[BN_MAX / 32][16], uint64_t adesc, uint64_t bdesc, bool accumulate) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
#pragma unroll
        for (int c = 0; c < NCH; ++c) {
            if constexpr (std::is_same_v<Acc, int32_t>) {
                tc::wgmma_m64n32k32_s8(acc[c], adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(c * 256 + 2 * k), accumulate || k != 0);
            } else if constexpr (FP8) {
                tc::wgmma_m64n32k32_e4m3(acc[c], adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(c * 256 + 2 * k), accumulate || k != 0);
            } else {
                tc::wgmma_m64n32k16(acc[c], adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(c * 256 + 2 * k), accumulate || k != 0);
            }
        }
    }
}

// ROWS: int8 operands with per-row factors (GemmDesc::row_scale), their own forms so that those without keep their code
template <int ACT, GemmType IN, GemmType OUT, bool ROWS>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tma_a,
                                                                     const __grid_constant__ CUtensorMap tma_w,
                                                                     const GemmKernelParams p) {
    constexpr bool FP8 = IN == GEMM_E4M3;
    constexpr bool S8 = IN == GEMM_S8;
    constexpr bool STORE_S8 = OUT == GEMM_S8;   // fp16 operands, int8 output
    constexpr int KB = FP8 || S8 ? BK8 : BK;   // K elements per block
    using Acc = std::conditional_t<S8, int32_t, float>;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // realign by an integer offset from the __shared__ symbol so the compiler keeps the shared address space
    uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
    const uint32_t a_bytes = BM * 128;
    const uint32_t w_bytes = (uint32_t)p.bn * 128;   // a multiple of 4 KB: every stage stays 1024-byte aligned
    const uint32_t stage_bytes = a_bytes + w_bytes;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * stage_bytes);
    uint64_t* empty = full + STAGES;
    const int nch = p.bn / 32;

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) {
            tc::mbar_init(&full[s], 1);
            tc::mbar_init(&empty[s], 2);   // one arrival per consumer warpgroup
        }
        tc::fence_barrier_init();
        tc::prefetch_tmap(&tma_a);
        tc::prefetch_tmap(&tma_w);
    }
    __syncthreads();
    const int wg = threadIdx.x >> 7;

    if (wg == 0) {
        if (threadIdx.x == 0) {
            int s = 0;
            uint32_t ph = 0;
            int mt, nt;
            for (int i = 0; gemm_tile_at(p, i, &mt, &nt); ++i) {
                const int batch = mt / p.tiles_per_batch;
                const int r0 = (mt % p.tiles_per_batch) * BM;
                for (int kb = 0; kb < p.num_k_blocks; ++kb) {
                    tc::mbar_wait_silent(&empty[s], ph ^ 1);
                    tc::mbar_arrive_expect_tx(&full[s], stage_bytes);
                    uint8_t* st = smem + s * stage_bytes;
                    tc::tma_load_3d(st, &tma_a, &full[s], kb * KB, r0, batch);
                    tc::tma_load_2d(st + a_bytes, &tma_w, &full[s], kb * KB, nt * p.bn);
                    if (++s == STAGES) {
                        s = 0;
                        ph ^= 1;
                    }
                }
            }
        }
        return;
    }

    const int half = wg - 1;                   // rows 64 * half .. + 63 of the tile
    const int t = threadIdx.x - 128 * wg;
    const int lane = t & 31, quad = lane & 3;
    const int rloc = half * 64 + (t >> 5) * 16 + (lane >> 2);   // tile rows rloc and rloc + 8
    const int n_out_total = ACT == GEMM_ACT_SWIGLU ? p.N / 2 : p.N;
    int s = 0;
    uint32_t ph = 0;
    int mt, nt;
    for (int ti = 0; gemm_tile_at(p, ti, &mt, &nt); ++ti) {
        Acc acc[BN_MAX / 32][16];
        int prev = -1;   // stage read by the wgmma group still in flight
        for (int kb = 0; kb < p.num_k_blocks; ++kb) {
            tc::mbar_wait_silent(&full[s], ph);
            const uint32_t st = tc::smem_u32(smem + s * stage_bytes);
            const uint64_t adesc = tc::wgmma_desc_sw128(st + (uint32_t)(half * 64 * 128));
            const uint64_t bdesc = tc::wgmma_desc_sw128(st + a_bytes);
            tc::wgmma_fence();
            switch (nch) {   // the chunk count as a constant: no predicated wgmma, no registers ptxas must fence
                case 1: wgmma_k_block<1, FP8>(acc, adesc, bdesc, kb != 0); break;
                case 2: wgmma_k_block<2, FP8>(acc, adesc, bdesc, kb != 0); break;
                case 3: wgmma_k_block<3, FP8>(acc, adesc, bdesc, kb != 0); break;
                default: wgmma_k_block<4, FP8>(acc, adesc, bdesc, kb != 0); break;
            }
            tc::wgmma_commit();
            // one group stays in flight: the previous K block's group has completed, so its stage goes back to the producer
            tc::wgmma_wait<1>();
            if (prev >= 0 && t == 0) tc::mbar_arrive(&empty[prev]);
            prev = s;
            if (++s == STAGES) {
                s = 0;
                ph ^= 1;
            }
        }
        tc::wgmma_wait<0>();
        if (t == 0) tc::mbar_arrive(&empty[prev]);

        // ---- epilogue from the accumulator fragments: rows rloc (+ 8), columns 32 c + 8 j + 2 quad (+ 1)
        const int batch = mt / p.tiles_per_batch;
        const int r0 = (mt % p.tiles_per_batch) * BM;
        const int n0 = nt * p.bn;
        // 32-bit division only: a 64-bit division is a library call, and a call in this function makes ptxas serialise the
        // wgmma pipeline.  make_gemm_plan checks that rows and the output blocking fit in 32 bits.
        bool valid[2];
        long long g[2], off[2];
        float r_a[2], r_res[2];
        float r_q[2];   // int8 operands with row factors: the A row's dequantisation factor (GemmDesc::row_scale)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = r0 + rloc + 8 * h;
            valid[h] = row < p.rows_per_batch;
            const uint32_t g32 = (uint32_t)(batch * p.rows_per_batch + row);
            g[h] = g32;
            off[h] = valid[h] ? (long long)(g32 / p.out_m1) * p.out_s0 + (long long)(g32 % p.out_m1) * p.out_s1 : 0;
            if constexpr (ROWS) {
                r_q[h] = valid[h] ? __ldg(p.row_scale + g[h]) : 0.0f;
            }
            // folded RMSNorm: 1/rms of this row of A and of the residual row, from the partial sums of squares (fixed order)
            r_a[h] = 1.0f;
            r_res[h] = 1.0f;
            if (p.a_ss && valid[h]) {
                float ss = 0.0f;
                for (int i = 0; i < p.a_ss_parts; ++i) ss += __ldg(p.a_ss + g[h] * p.a_ss_parts + i);
                r_a[h] = rsqrtf(ss * p.norm_inv_dim + p.norm_eps);
            }
            if (p.res_ss && valid[h]) {
                float ss = 0.0f;
                for (int i = 0; i < p.res_ss_parts; ++i) ss += __ldg(p.res_ss + g[h] * p.res_ss_parts + i);
                r_res[h] = rsqrtf(ss * p.norm_inv_dim + p.norm_eps);
            }
        }
        if constexpr (S8 && ACT != GEMM_ACT_ROPE) {
            // s32 -> fp32 (cvt.rn) is exact up to |acc| = 2^24 (127^2 K < 2^24 up to K = 1024); beyond it rounds to nearest
            // even.  With row factors: v = (float(acc) * row) * col (+ bias), the second product fused with the bias.
#pragma unroll
            for (int c = 0; c < BN_MAX / 32; ++c) {
                if (c >= nch) continue;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int nc = n0 + c * 32 + 8 * j + 2 * quad;
                    const float2 sc = __ldg(reinterpret_cast<const float2*>(p.col_scale + nc));
                    float2 b2 = make_float2(0.0f, 0.0f);
                    if (p.bias) b2 = __ldg(reinterpret_cast<const float2*>(p.bias + nc));
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        if (!valid[h]) continue;
                        float v0, v1;
                        if constexpr (ROWS) {
                            v0 = fmaf(__fmul_rn((float)acc[c][4 * j + 2 * h], r_q[h]), sc.x, b2.x);
                            v1 = fmaf(__fmul_rn((float)acc[c][4 * j + 2 * h + 1], r_q[h]), sc.y, b2.y);
                        } else {
                            v0 = fmaf((float)acc[c][4 * j + 2 * h], sc.x, b2.x);
                            v1 = fmaf((float)acc[c][4 * j + 2 * h + 1], sc.y, b2.y);
                        }
                        *reinterpret_cast<__half2*>(p.out + off[h] + nc) = __floats2half2_rn(act_apply<ACT>(v0), act_apply<ACT>(v1));
                    }
                }
            }
        } else if constexpr (ACT == GEMM_ACT_ROPE) {
            // head_dim 64 = two 32-column chunks (x1 | x2): out1 = cos*x1 - sin*x2, out2 = sin*x1 + cos*x2
#pragma unroll
            for (int c = 0; c < BN_MAX / 32; c += 2) {
                if (c < nch) {
                    const int nc0 = n0 + c * 32;
                    const bool rot = nc0 < p.rope_cols;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        if (!valid[h]) continue;
                        const float4* tab = reinterpret_cast<const float4*>(p.rope) + (int)((uint32_t)g[h] % (uint32_t)p.rope_T);
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const int col = 8 * j + 2 * quad;   // column pair (col, col + 1) of x1; x2 is 32 columns on
                            float a0, a1, b0, b1;
                            if constexpr (S8) {
                                // (float(acc) * row factor) * column factor, in that order
                                const float2 ca = __ldg(reinterpret_cast<const float2*>(p.col_scale + nc0 + col));
                                const float2 cb = __ldg(reinterpret_cast<const float2*>(p.col_scale + nc0 + 32 + col));
                                a0 = __fmul_rn(__fmul_rn(__int2float_rn(acc[c][4 * j + 2 * h]), r_q[h]), ca.x);
                                a1 = __fmul_rn(__fmul_rn(__int2float_rn(acc[c][4 * j + 2 * h + 1]), r_q[h]), ca.y);
                                b0 = __fmul_rn(__fmul_rn(__int2float_rn(acc[c + 1][4 * j + 2 * h]), r_q[h]), cb.x);
                                b1 = __fmul_rn(__fmul_rn(__int2float_rn(acc[c + 1][4 * j + 2 * h + 1]), r_q[h]), cb.y);
                            } else {
                                a0 = acc[c][4 * j + 2 * h] * r_a[h];
                                a1 = acc[c][4 * j + 2 * h + 1] * r_a[h];
                                b0 = acc[c + 1][4 * j + 2 * h] * r_a[h];
                                b1 = acc[c + 1][4 * j + 2 * h + 1] * r_a[h];
                            }
                            if (rot) {
                                const float4 cs = __ldg(tab + (size_t)(col / 2) * p.rope_stride);
                                const float x0 = cs.x * a0 - cs.y * b0, y0 = cs.y * a0 + cs.x * b0;
                                const float x1 = cs.z * a1 - cs.w * b1, y1 = cs.w * a1 + cs.z * b1;
                                a0 = x0; b0 = y0; a1 = x1; b1 = y1;
                            }
                            *reinterpret_cast<__half2*>(p.out + off[h] + nc0 + col) = __floats2half2_rn(a0, a1);
                            *reinterpret_cast<__half2*>(p.out + off[h] + nc0 + 32 + col) = __floats2half2_rn(b0, b1);
                        }
                    }
                }
            }
        } else {
            float ss_out[2][BN_MAX / 32];   // sums of squares of what this thread stores, per row and 32-column chunk
#pragma unroll
            for (int c = 0; c < BN_MAX / 32; ++c) {
                ss_out[0][c] = ss_out[1][c] = 0.0f;
                if (c >= nch) continue;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int nc = n0 + c * 32 + 8 * j + 2 * quad;
                    float2 b2 = make_float2(0.0f, 0.0f);
                    if (p.bias) b2 = __ldg(reinterpret_cast<const float2*>(p.bias + nc));
                    float2 gain = make_float2(1.0f, 1.0f);
                    if (p.residual && p.res_gain) gain = __ldg(reinterpret_cast<const float2*>(p.res_gain + nc));
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        if (!valid[h]) continue;
                        float v0 = acc[c][4 * j + 2 * h] * r_a[h] + b2.x;
                        float v1 = acc[c][4 * j + 2 * h + 1] * r_a[h] + b2.y;
                        if constexpr (ACT == GEMM_ACT_SWIGLU) {
                            // columns (2i, 2i + 1) = (y, gate) -> output column i
                            if constexpr (FP8) {
                                reinterpret_cast<uint8_t*>(p.out)[off[h] + nc / 2] = (uint8_t)tc::cvt_e4m3x2(v0 * swish_fast(v1), 0.0f);
                            } else {
                                p.out[off[h] + nc / 2] = __float2half_rn(v0 * swish_fast(v1));
                            }
                        } else {
                            if (p.residual) {
                                const float2 f = __half22float2(
                                        *reinterpret_cast<const __half2*>(p.residual + g[h] * (long long)n_out_total + nc));
                                const float ar = p.alpha * r_res[h];
                                v0 += (ar * gain.x) * f.x;
                                v1 += (ar * gain.y) * f.y;
                            }
                            const __half2 o = __floats2half2_rn(act_apply<ACT>(v0), act_apply<ACT>(v1));
                            if (p.out_ss) {
                                const float2 f = __half22float2(o);
                                ss_out[h][c] = fmaf(f.x, f.x, ss_out[h][c]);
                                ss_out[h][c] = fmaf(f.y, f.y, ss_out[h][c]);
                            }
                            if constexpr (STORE_S8) {
                                const int32_t q0 = tc::cvt_rni_sat_s8(kInt8ActScale * act_apply<ACT>(v0));
                                const int32_t q1 = tc::cvt_rni_sat_s8(kInt8ActScale * act_apply<ACT>(v1));
                                *reinterpret_cast<uint16_t*>(reinterpret_cast<int8_t*>(p.out) + off[h] + nc) =
                                        (uint16_t)((q0 & 0xff) | ((q1 & 0xff) << 8));
                            } else {
                                *reinterpret_cast<__half2*>(p.out + off[h] + nc) = o;
                            }
                        }
                    }
                }
            }
            if (p.out_ss) {
                // one partial per (column tile, 32-column chunk): the four lanes of a quad hold a row's columns
#pragma unroll
                for (int h = 0; h < 2; ++h) {
#pragma unroll
                    for (int c = 0; c < GEMM_PARTS; ++c) {
                        float v = ss_out[h][c];
                        v += __shfl_xor_sync(0xffffffffu, v, 1);
                        v += __shfl_xor_sync(0xffffffffu, v, 2);
                        if (quad == 0 && valid[h]) p.out_ss[g[h] * (long long)(p.n_tiles * GEMM_PARTS) + nt * GEMM_PARTS + c] = v;
                    }
                }
            }
        }
    }
}

// Optional inputs of a kernel form's epilogue (GemmForm::reads)
enum : unsigned {
    READS_BIAS = 1,
    READS_RESIDUAL = 2,    // residual, res_gain, res_ss
    READS_A_SS = 4,
    READS_OUT_SS = 8,
    READS_COL_SCALE = 16,  // required by the forms that read it
};
constexpr unsigned READS_PLAIN = READS_BIAS | READS_RESIDUAL | READS_A_SS | READS_OUT_SS;

using GemmKernel = void (*)(CUtensorMap, CUtensorMap, GemmKernelParams);

// One built instantiation of gemm_wgmma_kernel: the descriptors it runs (types, activation, row_scale set or not) and the
// optional inputs its epilogue reads
struct GemmForm {
    GemmType in, out;
    int act;
    bool rows;
    unsigned reads;
    GemmKernel kernel;
};

template <int ACT, GemmType IN, GemmType OUT, bool ROWS = false>
GemmForm form(unsigned reads) {
    return {IN, OUT, ACT, ROWS, reads, gemm_wgmma_kernel<ACT, IN, OUT, ROWS>};
}

const GemmForm kForms[] = {
        form<GEMM_ACT_NONE, GEMM_F16, GEMM_F16>(READS_PLAIN),
        form<GEMM_ACT_SWISH, GEMM_F16, GEMM_F16>(READS_PLAIN),
        form<GEMM_ACT_SWISH_CLAMP, GEMM_F16, GEMM_F16>(READS_PLAIN),
        form<GEMM_ACT_TANH, GEMM_F16, GEMM_F16>(READS_PLAIN),
        form<GEMM_ACT_TANH_X5, GEMM_F16, GEMM_F16>(READS_PLAIN),
        form<GEMM_ACT_SWIGLU, GEMM_F16, GEMM_F16>(READS_BIAS | READS_A_SS),
        form<GEMM_ACT_ROPE, GEMM_F16, GEMM_F16>(READS_A_SS),
        form<GEMM_ACT_TANH, GEMM_F16, GEMM_S8>(READS_BIAS),
        form<GEMM_ACT_NONE, GEMM_E4M3, GEMM_F16>(READS_PLAIN),
        form<GEMM_ACT_SWIGLU, GEMM_E4M3, GEMM_E4M3>(READS_BIAS | READS_A_SS),
        form<GEMM_ACT_NONE, GEMM_S8, GEMM_F16>(READS_COL_SCALE | READS_BIAS),
        form<GEMM_ACT_TANH_X5, GEMM_S8, GEMM_F16>(READS_COL_SCALE | READS_BIAS),
        form<GEMM_ACT_NONE, GEMM_S8, GEMM_F16, true>(READS_COL_SCALE | READS_BIAS),
        form<GEMM_ACT_ROPE, GEMM_S8, GEMM_F16, true>(READS_COL_SCALE),
};

int elem_bytes(GemmType t) { return t == GEMM_F16 ? 2 : 1; }

std::string type_name(GemmType t) {
    return t == GEMM_F16 ? "fp16" : t == GEMM_E4M3 ? "E4M3" : t == GEMM_S8 ? "int8" : "type " + std::to_string((int)t);
}

// The descriptor's form, and every input it sets that the form does not read (or col_scale missing where it is required)
const GemmForm& find_form(const GemmDesc& d) {
    const std::string what = type_name(d.in_type) + " operands, " + type_name(d.out_type) + " output, activation " +
                             std::to_string(d.act) + (d.row_scale ? " and row factors" : "");
    const GemmForm* f = std::find_if(std::begin(kForms), std::end(kForms), [&](const GemmForm& e) {
        return e.in == d.in_type && e.out == d.out_type && e.act == d.act && e.rows == (d.row_scale != nullptr);
    });
    if (f == std::end(kForms)) throw std::invalid_argument("gemm: no kernel form for " + what);
    const std::pair<unsigned, const char*> inputs[] = {
            {d.bias ? READS_BIAS : 0u, "bias"}, {d.residual || d.res_gain || d.res_ss ? READS_RESIDUAL : 0u, "residual"},
            {d.a_ss ? READS_A_SS : 0u, "a_ss"}, {d.out_ss ? READS_OUT_SS : 0u, "out_ss"},
            {d.col_scale ? READS_COL_SCALE : 0u, "col_scale"}};
    for (const auto& [given, name] : inputs) {
        if (given & ~f->reads) throw std::invalid_argument(std::string("gemm: the form for ") + what + " takes no " + name);
    }
    if ((f->reads & READS_COL_SCALE) && !d.col_scale) throw std::invalid_argument("gemm: the form for " + what + " needs col_scale");
    return *f;
}

using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                              const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeFn get_encode_fn() {
    // function-local static: initialised once, thread-safe (runners are created concurrently)
    static const EncodeFn fn = [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        B200_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
        if (q != cudaDriverEntryPointSuccess || !p) throw CudaError("cuTensorMapEncodeTiled entry point not available");
        return reinterpret_cast<EncodeFn>(p);
    }();
    return fn;
}

CUtensorMap encode(const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                   const cuuint32_t* box, CUtensorMapSwizzle swz, uint32_t elem_bytes) {
    CUtensorMap m;
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    const CUtensorMapDataType dt = elem_bytes == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    const CUresult r = get_encode_fn()(&m, dt, (cuuint32_t)rank, const_cast<void*>(base), dims,
                                       strides_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                                       CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        throw CudaError("cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r));
    }
    return m;
}

}  // namespace

CUtensorMap make_tmap_2d(const void* base, uint64_t inner, uint64_t outer, uint64_t outer_stride_bytes, uint32_t box_inner,
                         uint32_t box_outer, uint32_t elem_bytes) {
    const cuuint64_t dims[2] = {inner, outer};
    const cuuint64_t strides[1] = {outer_stride_bytes};
    const cuuint32_t box[2] = {box_inner, box_outer};
    const CUtensorMapSwizzle swz = box_inner * elem_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                   : box_inner * elem_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                                                  : CU_TENSOR_MAP_SWIZZLE_NONE;
    return encode(base, 2, dims, strides, box, swz, elem_bytes);
}

CUtensorMap make_tmap_3d(const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t s1_bytes, uint64_t s2_bytes,
                         uint32_t b0, uint32_t b1, uint32_t b2, uint32_t elem_bytes) {
    const cuuint64_t dims[3] = {d0, d1, d2};
    const cuuint64_t strides[2] = {s1_bytes, s2_bytes};
    const cuuint32_t box[3] = {b0, b1, b2};
    const CUtensorMapSwizzle swz = b0 * elem_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                   : b0 * elem_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                                           : CU_TENSOR_MAP_SWIZZLE_NONE;
    return encode(base, 3, dims, strides, box, swz, elem_bytes);
}

static int pick_bn(int N) {
    // largest tile width <= BN_MAX that divides N and is a multiple of 32
    for (int bn = BN_MAX; bn >= 32; bn -= 32) {
        if (N % bn == 0) return bn;
    }
    return 0;
}

int gemm_out_ss_parts(int N) {
    const int bn = pick_bn(N);
    if (bn <= 0) throw std::invalid_argument("gemm: N must be a multiple of 32");
    return (N / bn) * GEMM_PARTS;
}

namespace {

// Everything make_gemm_plan checks and decides, on the host alone (no driver call): the form, the tile width, the grid,
// the shared memory.  The tensor maps are left to make_gemm_plan.
GemmPlan plan_gemm(const GemmDesc& d) {
    const GemmForm& f = find_form(d);
    const int eb = elem_bytes(d.in_type);   // bytes per A / W element
    const int kb = 128 / eb;                // elements per K block: one 128-byte swizzle row
    if (d.K % kb != 0 || d.K <= 0) {
        throw std::invalid_argument(eb == 1 ? "gemm: E4M3 / int8 K must be a positive multiple of 128" : "gemm: K must be a positive multiple of 64");
    }
    if (d.N % 32 != 0) throw std::invalid_argument("gemm: N must be a multiple of 32");
    if (d.batches < 1 || d.rows_per_batch < 1) throw std::invalid_argument("gemm: empty A");
    if ((d.a_row_stride * eb) % 16 != 0 || (d.a_batch_stride * eb) % 16 != 0) {
        throw std::invalid_argument("gemm: A strides must be multiples of 16 bytes");
    }
    GemmPlan p{};
    p.d = d;
    p.kernel = reinterpret_cast<const void*>(f.kernel);
    p.num_k_blocks = d.K / kb;
    p.bn = pick_bn(d.N);
    // few row tiles: split N further to fill more SMs.  Not with out_ss, whose partial slots are laid out for tiles of
    // pick_bn(N) columns (gemm_out_ss_parts); the tile width only changes the occupancy.
    if (!d.out_ss && d.N / p.bn < 2 && d.N >= 128 && (long long)d.batches * ((d.rows_per_batch + BM - 1) / BM) < kNumSMs / 2) {
        p.bn = pick_bn(d.N / 2);
    }
    if (p.bn == 0) throw std::invalid_argument("gemm: no valid tile width");
    if (d.out_ss) {
        // every 32-column chunk of every column tile owns one partial slot
        if (p.bn != pick_bn(d.N) || p.bn / 32 != GEMM_PARTS || d.act == GEMM_ACT_SWIGLU || d.act == GEMM_ACT_ROPE) {
            throw std::invalid_argument("gemm: out_ss needs a plain epilogue and tiles of 128 columns");
        }
    }
    if ((d.a_ss && (d.a_ss_parts < 1 || d.norm_dim < 1)) || (d.res_ss && (d.res_ss_parts < 1 || d.norm_dim < 1 || !d.residual))) {
        throw std::invalid_argument("gemm: folded RMSNorm needs the partial count, the norm dimension and a residual");
    }
    if (d.act == GEMM_ACT_SWIGLU && (p.bn % 64) != 0) throw std::invalid_argument("gemm: swiglu needs BN % 64 == 0");
    if (d.act == GEMM_ACT_ROPE && ((p.bn % 64) != 0 || !d.rope || d.rope_T <= 0)) {
        throw std::invalid_argument("gemm: rope epilogue needs BN % 64 == 0 and a table");
    }
    p.tiles_per_batch = (d.rows_per_batch + BM - 1) / BM;
    if ((long long)p.tiles_per_batch * BM * d.batches >= (1LL << 31) || d.out_m1 < 1 || d.out_m1 >= (1LL << 32)) {
        throw std::invalid_argument("gemm: rows and output blocking must fit 32-bit index arithmetic");
    }
    p.grid = dim3((unsigned)(p.tiles_per_batch * d.batches), (unsigned)(d.N / p.bn), 1);
    p.smem = (size_t)STAGES * ((size_t)BM * 128 + (size_t)p.bn * 128) + 256 + 1024;
    if (p.smem > 227 * 1024) throw std::logic_error("gemm: shared-memory plan does not fit");
    return p;
}

}  // namespace

GemmPlan make_gemm_plan(const GemmDesc& d) {
    GemmPlan p = plan_gemm(d);
    const uint32_t eb = elem_bytes(d.in_type), kb = 128 / eb;
    const uint64_t batch_stride = d.batches > 1 ? (uint64_t)d.a_batch_stride * eb : (uint64_t)d.a_row_stride * eb * d.rows_per_batch;
    p.tma_a = make_tmap_3d(d.a, (uint64_t)(d.a_inner > 0 ? d.a_inner : d.K), (uint64_t)d.rows_per_batch, (uint64_t)d.batches, (uint64_t)d.a_row_stride * eb,
                           batch_stride, kb, BM, 1, eb);
    p.tma_w = make_tmap_2d(d.w, (uint64_t)d.K, (uint64_t)d.N, (uint64_t)d.K * eb, kb, (uint32_t)p.bn, eb);
    return p;
}

void run_gemm(const GemmPlan& p, cudaStream_t stream) {
    GemmKernelParams k{};
    k.rows_per_batch = p.d.rows_per_batch;
    k.tiles_per_batch = p.tiles_per_batch;
    k.N = p.d.N;
    k.num_k_blocks = p.num_k_blocks;
    k.bn = p.bn;
    k.bias = p.d.bias;
    k.out = static_cast<__half*>(p.d.out);
    k.out_m1 = (uint32_t)p.d.out_m1;
    k.out_s0 = p.d.out_s0;
    k.out_s1 = p.d.out_s1;
    k.rope = p.d.rope;
    k.rope_T = p.d.rope_T;
    k.rope_cols = p.d.rope_cols;
    k.rope_stride = p.d.rope_stride;
    k.residual = p.d.residual;
    k.alpha = p.d.alpha;
    k.n_tiles = p.d.N / p.bn;
    k.m_tiles = p.tiles_per_batch * p.d.batches;
    k.num_tiles = k.m_tiles * k.n_tiles;
    k.mfast = k.m_tiles < k.n_tiles ? 1 : 0;
    k.out_ss = p.d.out_ss;
    k.a_ss = p.d.a_ss;
    k.res_ss = p.d.res_ss;
    k.res_gain = p.d.res_gain;
    k.a_ss_parts = p.d.a_ss_parts;
    k.res_ss_parts = p.d.res_ss_parts;
    k.norm_inv_dim = p.d.norm_dim > 0 ? 1.0f / (float)p.d.norm_dim : 0.0f;
    k.norm_eps = p.d.norm_eps;
    k.col_scale = p.d.col_scale;
    k.row_scale = p.d.row_scale;
    const int max_ctas = p.d.max_ctas > 0 && p.d.max_ctas < kNumSMs ? p.d.max_ctas : kNumSMs;
    const int grid = k.num_tiles < max_ctas ? k.num_tiles : max_ctas;
    ensure_dynamic_smem(p.kernel, 227 * 1024);
    reinterpret_cast<GemmKernel>(p.kernel)<<<grid, GEMM_THREADS, p.smem, stream>>>(p.tma_a, p.tma_w, k);
    B200_CUDA(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------
// test hook: host buffers in, host buffer out
// ------------------------------------------------------------------------------------------------
namespace {

// Refuses, before anything is allocated, a descriptor that would make the kernel read or write outside a buffer of the
// lengths given (b200_gemm_test_desc; lengths in elements of each buffer's type).  Ranges first: with rows < 2^31 and
// strides and offsets < 2^30, every sum below stays under 2^62.
void check_gemm_test_desc(const b200_gemm_test_desc& t) {
    auto need = [](bool ok, const char* what) {
        if (!ok) throw std::invalid_argument(std::string("b200_test_gemm_desc: ") + what);
    };
    constexpr int64_t kMax = 1LL << 30;
    need(t.in_type >= GEMM_F16 && t.in_type <= GEMM_S8 && t.out_type >= GEMM_F16 && t.out_type <= GEMM_S8, "unknown element type");
    need(t.batches >= 1 && t.rows_per_batch >= 1 && (int64_t)t.batches * t.rows_per_batch < (1LL << 31), "rows out of range");
    need(t.K >= 1 && t.K <= (1 << 16) && t.N >= 1 && t.N <= (1 << 16), "K or N out of range");
    need(t.a_inner >= 0 && t.a_inner <= t.K, "a_inner must lie in [0, K]");
    need(t.a_row_stride >= 0 && t.a_row_stride < kMax && t.a_batch_stride >= 0 && t.a_batch_stride < kMax, "A strides out of range");
    need(t.out_offset >= 0 && t.out_offset < kMax && t.out_m1 >= 1 && t.out_m1 < kMax && t.out_s0 >= 0 && t.out_s0 < kMax &&
                 t.out_s1 >= 0 && t.out_s1 < kMax, "output addressing out of range");
    // the epilogue stores column pairs as one __half2 (two bytes with the int8 output)
    need(t.out_offset % 2 == 0 && t.out_s0 % 2 == 0 && t.out_s1 % 2 == 0, "output offset and strides must be even");
    need(t.a_ss_parts >= 0 && t.a_ss_parts <= 4096 && t.res_ss_parts >= 0 && t.res_ss_parts <= 4096, "partial counts out of range");
    need(t.a_len >= 0 && t.w_len >= 0 && t.bias_len >= 0 && t.residual_len >= 0 && t.res_gain_len >= 0 && t.a_ss_len >= 0 &&
                 t.res_ss_len >= 0 && t.out_len >= 0 && t.out_ss_len >= 0 && t.col_scale_len >= 0 && t.row_scale_len >= 0,
         "negative buffer length");
    need(t.a && t.w && t.out, "A, W and out are required");
    const int64_t rows = (int64_t)t.batches * t.rows_per_batch;
    // A: the tensor map's extent, (a_inner or K) x rows_per_batch x batches; TMA reads nothing beyond it
    const int64_t inner = t.a_inner > 0 ? t.a_inner : t.K;
    need((t.batches - 1) * t.a_batch_stride + (int64_t)(t.rows_per_batch - 1) * t.a_row_stride + inner <= t.a_len, "A is too short");
    need((int64_t)t.N * t.K <= t.w_len, "W is too short");
    need(!t.bias || t.N <= t.bias_len, "bias is too short");
    need(!t.col_scale || t.N <= t.col_scale_len, "col_scale is too short");
    need(!t.row_scale || rows <= t.row_scale_len, "row_scale is too short");
    // out: the largest row offset over g < rows, with non-negative strides at the last g or at the last g of the previous
    // out_m1 block
    const int64_t q = (rows - 1) / t.out_m1, r = (rows - 1) % t.out_m1;
    int64_t last_row = q * t.out_s0 + r * t.out_s1;
    if (q > 0) last_row = std::max(last_row, (q - 1) * t.out_s0 + (t.out_m1 - 1) * t.out_s1);
    const int n_out = t.act == GEMM_ACT_SWIGLU ? t.N / 2 : t.N;
    need(t.out_offset + last_row + n_out <= t.out_len, "out is too short");
    // the residual is addressed as g * N + n whatever the output strides
    need(!t.residual || rows * t.N <= t.residual_len, "residual is too short");
    need(!t.res_gain || t.N <= t.res_gain_len, "res_gain is too short");
    need(!t.a_ss || rows * t.a_ss_parts <= t.a_ss_len, "a_ss is too short");
    need(!t.res_ss || rows * t.res_ss_parts <= t.res_ss_len, "res_ss is too short");
    need(!t.out_ss || rows * (t.N / 32) <= t.out_ss_len, "out_ss is too short");
    if (t.act == GEMM_ACT_ROPE) {
        // the table has max_seq_len positions per dim pair, and the kernel reads position g % rope_T
        need(t.theta > 0.0f && t.max_seq_len >= 1 && t.max_seq_len <= (1 << 16) && t.rope_T >= 1 && t.rope_T <= t.max_seq_len,
             "RoPE needs theta > 0 and 1 <= rope_T <= max_seq_len");
    }
}

}  // namespace

void test_gemm_desc_host(int device, const b200_gemm_test_desc& t) {
    check_gemm_test_desc(t);
    const int64_t rows = (int64_t)t.batches * t.rows_per_batch;
    const std::vector<float> rope = t.act == GEMM_ACT_ROPE ? rope_table(t.theta, t.max_seq_len) : std::vector<float>();
    // the descriptor on the host buffers first: every refusal of make_gemm_plan comes before any device work
    GemmDesc d{};
    d.in_type = (GemmType)t.in_type;
    d.out_type = (GemmType)t.out_type;
    d.col_scale = t.col_scale;
    d.row_scale = t.row_scale;
    d.a = t.a;
    d.batches = t.batches;
    d.rows_per_batch = t.rows_per_batch;
    d.a_row_stride = t.a_row_stride;
    d.a_batch_stride = t.a_batch_stride;
    d.a_inner = t.a_inner;
    d.w = t.w;
    d.N = t.N;
    d.K = t.K;
    d.bias = t.bias;
    d.act = t.act;
    d.out = t.out;
    d.out_m1 = t.out_m1;
    d.out_s0 = t.out_s0;
    d.out_s1 = t.out_s1;
    if (t.act == GEMM_ACT_ROPE) {
        d.rope = rope.data();
        d.rope_T = t.rope_T;
        d.rope_cols = t.rope_cols;
        d.rope_stride = t.max_seq_len;
    }
    d.max_ctas = t.max_ctas;
    d.residual = reinterpret_cast<const __half*>(t.residual);
    d.alpha = t.alpha;
    d.out_ss = t.out_ss;
    d.a_ss = t.a_ss;
    d.a_ss_parts = t.a_ss_parts;
    d.res_ss = t.res_ss;
    d.res_ss_parts = t.res_ss_parts;
    d.res_gain = t.res_gain;
    d.norm_dim = t.norm_dim;
    d.norm_eps = t.norm_eps;
    plan_gemm(d);
    require_sm90(device);
    const size_t ei = elem_bytes(d.in_type), eo = elem_bytes(d.out_type);
    auto bytes = [](int64_t n, size_t elem) { return (size_t)(n > 0 ? n : 1) * elem; };
    uint8_t *d_a = nullptr, *d_w = nullptr, *d_out = nullptr;
    __half* d_res = nullptr;
    float *d_bias = nullptr, *d_gain = nullptr, *d_a_ss = nullptr, *d_res_ss = nullptr, *d_out_ss = nullptr, *d_rope = nullptr;
    float *d_col = nullptr, *d_row = nullptr;
    Arena arena;
    arena.allocate([&](Bump& b) {
        d_a = b.take<uint8_t>(bytes(t.a_len, ei));
        d_w = b.take<uint8_t>(bytes(t.w_len, ei));
        d_bias = b.take<float>(bytes(t.bias_len, 4));
        d_res = b.take<__half>(bytes(t.residual_len, 2));
        d_gain = b.take<float>(bytes(t.res_gain_len, 4));
        d_a_ss = b.take<float>(bytes(t.a_ss_len, 4));
        d_res_ss = b.take<float>(bytes(t.res_ss_len, 4));
        d_out = b.take<uint8_t>(bytes(t.out_len, eo));
        d_out_ss = b.take<float>(bytes(t.out_ss_len, 4));
        d_rope = b.take<float>(bytes((int64_t)rope.size(), 4));
        d_col = b.take<float>(bytes(t.col_scale_len, 4));
        d_row = b.take<float>(bytes(t.row_scale_len, 4));
    });
    auto up = [](void* dst, const void* src, int64_t n, size_t elem) {
        if (src && n > 0) B200_CUDA(cudaMemcpy(dst, src, (size_t)n * elem, cudaMemcpyHostToDevice));
    };
    up(d_a, t.a, t.a_len, ei);
    up(d_w, t.w, t.w_len, ei);
    up(d_bias, t.bias, t.bias_len, 4);
    up(d_res, t.residual, t.residual_len, 2);
    up(d_gain, t.res_gain, t.res_gain_len, 4);
    up(d_a_ss, t.a_ss, t.a_ss_len, 4);
    up(d_res_ss, t.res_ss, t.res_ss_len, 4);
    up(d_out, t.out, t.out_len, eo);
    up(d_rope, rope.data(), (int64_t)rope.size(), 4);
    up(d_col, t.col_scale, t.col_scale_len, 4);
    up(d_row, t.row_scale, t.row_scale_len, 4);
    if (t.out_ss) B200_CUDA(cudaMemset(d_out_ss, 0xff, bytes(t.out_ss_len, 4)));   // NaN: a partial never written shows
    // the same descriptor on the device copies
    d.a = d_a;
    d.w = d_w;
    d.out = d_out + t.out_offset * eo;
    if (d.rope) d.rope = d_rope;
    if (d.bias) d.bias = d_bias;
    if (d.residual) d.residual = d_res;
    if (d.res_gain) d.res_gain = d_gain;
    if (d.a_ss) d.a_ss = d_a_ss;
    if (d.res_ss) d.res_ss = d_res_ss;
    if (d.out_ss) d.out_ss = d_out_ss;
    if (d.col_scale) d.col_scale = d_col;
    if (d.row_scale) d.row_scale = d_row;
    const GemmPlan plan = make_gemm_plan(d);
    run_gemm(plan, nullptr);
    B200_CUDA(cudaDeviceSynchronize());
    B200_CUDA(cudaMemcpy(t.out, d_out, (size_t)t.out_len * eo, cudaMemcpyDeviceToHost));
    if (t.out_ss) B200_CUDA(cudaMemcpy(t.out_ss, d_out_ss, (size_t)rows * (t.N / 32) * 4, cudaMemcpyDeviceToHost));
}

}  // namespace b200
