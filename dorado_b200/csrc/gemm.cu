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
// A is addressed through a 3-D tensor map (k, row, batch) so that overlapping-row views work: the last conv of the LSTM
// models reads its im2col rows straight from the NTC activation buffer with row stride = stride * C_in (the reference's
// "cutlass_conv" trick, ConvStack.cpp:236-275).
#include "gemm.h"

#include "common.cuh"
#include "engine.h"

#include <cstdlib>
#include <cstring>
#include <vector>

namespace b200 {

namespace {

constexpr int BM = 128;
constexpr int BK = 64;
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
    uint32_t out_col_m1;
    long long out_col_s0;
    int bias_per_row;
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

// One K block (64) of a warpgroup's 64 x 32 NCH tile: 32 rows of W are 4 KB further on, 16 fp16 along K are +2 in the
// (addr >> 4) field of a descriptor.
template <int NCH>
__device__ __forceinline__ void wgmma_k_block(float (&acc)[BN_MAX / 32][16], uint64_t adesc, uint64_t bdesc, bool accumulate) {
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) {
#pragma unroll
        for (int c = 0; c < NCH; ++c) {
            tc::wgmma_m64n32k16(acc[c], adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(c * 256 + 2 * k), accumulate || k != 0);
        }
    }
}

template <int ACT>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_f16_wgmma_kernel(const __grid_constant__ CUtensorMap tma_a,
                                                                         const __grid_constant__ CUtensorMap tma_w,
                                                                         const GemmKernelParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // realign by an integer offset from the __shared__ symbol so the compiler keeps the shared address space
    uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
    const uint32_t a_bytes = BM * BK * 2;
    const uint32_t w_bytes = (uint32_t)p.bn * BK * 2;   // a multiple of 4 KB: every stage stays 1024-byte aligned
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
                    tc::tma_load_3d(st, &tma_a, &full[s], kb * BK, r0, batch);
                    tc::tma_load_2d(st + a_bytes, &tma_w, &full[s], kb * BK, nt * p.bn);
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
        float acc[BN_MAX / 32][16];
        int prev = -1;   // stage read by the wgmma group still in flight
        for (int kb = 0; kb < p.num_k_blocks; ++kb) {
            tc::mbar_wait_silent(&full[s], ph);
            const uint32_t st = tc::smem_u32(smem + s * stage_bytes);
            const uint64_t adesc = tc::wgmma_desc_sw128(st + (uint32_t)(half * 64 * 128));
            const uint64_t bdesc = tc::wgmma_desc_sw128(st + a_bytes);
            tc::wgmma_fence();
            switch (nch) {   // the chunk count as a constant: no predicated wgmma, no registers ptxas must fence
                case 1: wgmma_k_block<1>(acc, adesc, bdesc, kb != 0); break;
                case 2: wgmma_k_block<2>(acc, adesc, bdesc, kb != 0); break;
                case 3: wgmma_k_block<3>(acc, adesc, bdesc, kb != 0); break;
                default: wgmma_k_block<4>(acc, adesc, bdesc, kb != 0); break;
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
        // wgmma pipeline.  make_gemm_plan checks that rows, strides and column blocking fit in 32 bits.
        bool valid[2];
        long long g[2], off[2];
        float r_a[2], r_res[2], row_bias[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = r0 + rloc + 8 * h;
            valid[h] = row < p.rows_per_batch;
            const uint32_t g32 = (uint32_t)(batch * p.rows_per_batch + row);
            g[h] = g32;
            off[h] = valid[h] ? (long long)(g32 / p.out_m1) * p.out_s0 + (long long)(g32 % p.out_m1) * p.out_s1 : 0;
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
            row_bias[h] = (p.bias && p.bias_per_row && valid[h]) ? __ldg(p.bias + g[h]) : 0.0f;
        }
        if constexpr (ACT == GEMM_ACT_ROPE) {
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
                            float a0 = acc[c][4 * j + 2 * h] * r_a[h], a1 = acc[c][4 * j + 2 * h + 1] * r_a[h];
                            float b0 = acc[c + 1][4 * j + 2 * h] * r_a[h], b1 = acc[c + 1][4 * j + 2 * h + 1] * r_a[h];
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
                    if (p.bias && !p.bias_per_row) b2 = __ldg(reinterpret_cast<const float2*>(p.bias + nc));
                    float2 gain = make_float2(1.0f, 1.0f);
                    if (p.residual && p.res_gain) gain = __ldg(reinterpret_cast<const float2*>(p.res_gain + nc));
                    const long long coff = p.out_col_m1 > 0
                            ? (long long)((uint32_t)nc / p.out_col_m1) * p.out_col_s0 + (long long)((uint32_t)nc % p.out_col_m1)
                            : nc;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        if (!valid[h]) continue;
                        float v0 = acc[c][4 * j + 2 * h] * r_a[h] + b2.x + row_bias[h];
                        float v1 = acc[c][4 * j + 2 * h + 1] * r_a[h] + b2.y + row_bias[h];
                        if constexpr (ACT == GEMM_ACT_SWIGLU) {
                            // columns (2i, 2i + 1) = (y, gate) -> output column i
                            p.out[off[h] + nc / 2] = __float2half_rn(v0 * swish_fast(v1));
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
                            *reinterpret_cast<__half2*>(p.out + off[h] + coff) = o;
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
                   const cuuint32_t* box, CUtensorMapSwizzle swz) {
    CUtensorMap m;
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    const CUresult r = get_encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(base), dims,
                                       strides_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                                       CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        throw CudaError("cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r));
    }
    return m;
}

}  // namespace

CUtensorMap make_tmap_2d(const void* base, uint64_t inner, uint64_t outer, uint64_t outer_stride_bytes, uint32_t box_inner,
                         uint32_t box_outer) {
    const cuuint64_t dims[2] = {inner, outer};
    const cuuint64_t strides[1] = {outer_stride_bytes};
    const cuuint32_t box[2] = {box_inner, box_outer};
    const CUtensorMapSwizzle swz = box_inner * 2 == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                   : box_inner * 2 == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                                         : CU_TENSOR_MAP_SWIZZLE_NONE;
    return encode(base, 2, dims, strides, box, swz);
}

CUtensorMap make_tmap_3d(const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t s1_bytes, uint64_t s2_bytes,
                         uint32_t b0, uint32_t b1, uint32_t b2) {
    const cuuint64_t dims[3] = {d0, d1, d2};
    const cuuint64_t strides[2] = {s1_bytes, s2_bytes};
    const cuuint32_t box[3] = {b0, b1, b2};
    const CUtensorMapSwizzle swz = b0 * 2 == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                   : b0 * 2 == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                                  : CU_TENSOR_MAP_SWIZZLE_NONE;
    return encode(base, 3, dims, strides, box, swz);
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

GemmPlan make_gemm_plan(const GemmDesc& d) {
    if (d.K % BK != 0 || d.K <= 0) throw std::invalid_argument("gemm: K must be a positive multiple of 64");
    if (d.N % 32 != 0) throw std::invalid_argument("gemm: N must be a multiple of 32");
    if (d.batches < 1 || d.rows_per_batch < 1) throw std::invalid_argument("gemm: empty A");
    if ((d.a_row_stride * 2) % 16 != 0 || (d.a_batch_stride * 2) % 16 != 0) {
        throw std::invalid_argument("gemm: A strides must be multiples of 16 bytes");
    }
    GemmPlan p{};
    p.d = d;
    p.bn = pick_bn(d.N);
    if (d.N / p.bn < 2 && d.N >= 128 && (long long)d.batches * ((d.rows_per_batch + BM - 1) / BM) < kNumSMs / 2) {
        p.bn = pick_bn(d.N / 2);  // few row tiles: split N further to fill more SMs
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
    if ((long long)p.tiles_per_batch * BM * d.batches >= (1LL << 31) || d.out_m1 < 1 || d.out_m1 >= (1LL << 32) ||
        d.out_col_m1 < 0 || d.out_col_m1 >= (1LL << 32)) {
        throw std::invalid_argument("gemm: rows and output blocking must fit 32-bit index arithmetic");
    }
    p.grid = dim3((unsigned)(p.tiles_per_batch * d.batches), (unsigned)(d.N / p.bn), 1);
    p.smem = (size_t)STAGES * ((size_t)BM * BK * 2 + (size_t)p.bn * BK * 2) + 256 + 1024;
    if (p.smem > 227 * 1024) throw std::logic_error("gemm: shared-memory plan does not fit");
    const uint64_t batch_stride = d.batches > 1 ? (uint64_t)d.a_batch_stride * 2 : (uint64_t)d.a_row_stride * 2 * d.rows_per_batch;
    p.tma_a = make_tmap_3d(d.a, (uint64_t)(d.a_inner > 0 ? d.a_inner : d.K), (uint64_t)d.rows_per_batch, (uint64_t)d.batches, (uint64_t)d.a_row_stride * 2,
                           batch_stride, BK, BM, 1);
    p.tma_w = make_tmap_2d(d.w, (uint64_t)d.K, (uint64_t)d.N, (uint64_t)d.K * 2, BK, (uint32_t)p.bn);
    return p;
}

template <int ACT>
static void launch_gemm(int grid, size_t smem, cudaStream_t stream, const CUtensorMap& a, const CUtensorMap& w,
                        const GemmKernelParams& k) {
    ensure_dynamic_smem(gemm_f16_wgmma_kernel<ACT>, 227 * 1024);
    gemm_f16_wgmma_kernel<ACT><<<grid, GEMM_THREADS, smem, stream>>>(a, w, k);
}

void run_gemm(const GemmPlan& p, cudaStream_t stream) {
    GemmKernelParams k{};
    k.rows_per_batch = p.d.rows_per_batch;
    k.tiles_per_batch = p.tiles_per_batch;
    k.N = p.d.N;
    k.num_k_blocks = p.d.K / BK;
    k.bn = p.bn;
    k.bias = p.d.bias;
    k.out = p.d.out;
    k.out_m1 = (uint32_t)p.d.out_m1;
    k.out_s0 = p.d.out_s0;
    k.out_s1 = p.d.out_s1;
    k.out_col_m1 = (uint32_t)p.d.out_col_m1;
    k.out_col_s0 = p.d.out_col_s0;
    k.bias_per_row = p.d.bias_per_row;
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
    const int max_ctas = p.d.max_ctas > 0 && p.d.max_ctas < kNumSMs ? p.d.max_ctas : kNumSMs;
    const int grid = k.num_tiles < max_ctas ? k.num_tiles : max_ctas;
    switch (p.d.act) {
        case GEMM_ACT_NONE: launch_gemm<GEMM_ACT_NONE>(grid, p.smem, stream, p.tma_a, p.tma_w, k); break;
        case GEMM_ACT_SWISH: launch_gemm<GEMM_ACT_SWISH>(grid, p.smem, stream, p.tma_a, p.tma_w, k); break;
        case GEMM_ACT_SWISH_CLAMP: launch_gemm<GEMM_ACT_SWISH_CLAMP>(grid, p.smem, stream, p.tma_a, p.tma_w, k); break;
        case GEMM_ACT_TANH: launch_gemm<GEMM_ACT_TANH>(grid, p.smem, stream, p.tma_a, p.tma_w, k); break;
        case GEMM_ACT_TANH_X5: launch_gemm<GEMM_ACT_TANH_X5>(grid, p.smem, stream, p.tma_a, p.tma_w, k); break;
        case GEMM_ACT_SWIGLU: launch_gemm<GEMM_ACT_SWIGLU>(grid, p.smem, stream, p.tma_a, p.tma_w, k); break;
        case GEMM_ACT_ROPE: launch_gemm<GEMM_ACT_ROPE>(grid, p.smem, stream, p.tma_a, p.tma_w, k); break;
        default: throw std::invalid_argument("gemm: unknown activation");
    }
    B200_CUDA(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------
// test hook: host buffers in, host buffer out
// ------------------------------------------------------------------------------------------------
void test_gemm_host(int device, const uint16_t* a, const uint16_t* b, const float* bias, int M, int N, int K, int activation,
                    uint16_t* c) {
    require_sm90(device);
    const int Kp = (K + BK - 1) / BK * BK;
    const int n_out = activation == GEMM_ACT_SWIGLU ? N / 2 : N;
    Arena arena;
    arena.reserve((size_t)M * Kp * 2 + (size_t)N * Kp * 2 + (size_t)N * 4 + (size_t)M * n_out * 2 + 4096);
    auto* d_a = static_cast<__half*>(arena.take((size_t)M * Kp * 2));
    auto* d_w = static_cast<__half*>(arena.take((size_t)N * Kp * 2));
    auto* d_bias = static_cast<float*>(arena.take((size_t)N * 4));
    auto* d_c = static_cast<__half*>(arena.take((size_t)M * n_out * 2));
    B200_CUDA(cudaMemset(d_a, 0, (size_t)M * Kp * 2));
    B200_CUDA(cudaMemset(d_w, 0, (size_t)N * Kp * 2));
    B200_CUDA(cudaMemcpy2D(d_a, (size_t)Kp * 2, a, (size_t)K * 2, (size_t)K * 2, M, cudaMemcpyHostToDevice));
    B200_CUDA(cudaMemcpy2D(d_w, (size_t)Kp * 2, b, (size_t)K * 2, (size_t)K * 2, N, cudaMemcpyHostToDevice));
    if (bias) B200_CUDA(cudaMemcpy(d_bias, bias, (size_t)N * 4, cudaMemcpyHostToDevice));
    GemmDesc d{};
    d.a = d_a;
    d.batches = 1;
    d.rows_per_batch = M;
    d.a_row_stride = Kp;
    d.a_batch_stride = (int64_t)M * Kp;
    d.w = d_w;
    d.N = N;
    d.K = Kp;
    d.bias = bias ? d_bias : nullptr;
    d.act = activation;
    d.out = d_c;
    d.out_m1 = 1;
    d.out_s0 = n_out;
    d.out_s1 = 0;
    const GemmPlan plan = make_gemm_plan(d);
    run_gemm(plan, nullptr);
    B200_CUDA(cudaDeviceSynchronize());
    B200_CUDA(cudaMemcpy(c, d_c, (size_t)M * n_out * 2, cudaMemcpyDeviceToHost));
}

}  // namespace b200
