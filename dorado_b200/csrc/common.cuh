// Shared helpers for the sm_90a kernels of the basecalling engine.
#pragma once

#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <stdexcept>
#include <string>

namespace b200 {

struct CudaError : std::runtime_error {
    using std::runtime_error::runtime_error;
};

inline void cuda_check(cudaError_t e, const char* what, const char* file, int line) {
    if (e != cudaSuccess) {
        throw CudaError(std::string(what) + ": " + cudaGetErrorString(e) + " (" + file + ":" + std::to_string(line) + ")");
    }
}
#define B200_CUDA(expr) ::b200::cuda_check((expr), #expr, __FILE__, __LINE__)

constexpr int kNumSMs = 132;   // H100 SXM

// exact warp-wide max of finite floats in one redux.sync: order-preserving float <-> uint32 key
__device__ __forceinline__ float warp_max(float v) {
    const uint32_t u = __float_as_uint(v);
    const uint32_t key = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    const uint32_t m = __reduce_max_sync(0xffffffffu, key);
    return __uint_as_float((m & 0x80000000u) ? (m & 0x7fffffffu) : ~m);
}

// Activations on the SFU: one ex2 and one rcp each (MUFU.EX2 / MUFU.RCP, ~1 ulp), no IEEE division sequences.  Finite inputs
// only: e^x = inf gives the correct limit, x = -inf itself would give swish = NaN.
// tanh_mufu is MUFU.TANH (tanh.approx.f32, relative error ~2^-11).  It serves the LSTM gates (lstm_model.cu: the recurrences
// are SFU- and issue-bound and the score error is unchanged).  Swish through it -- h + h tanh(h), h = v / 2 -- was measured
// and REJECTED (battery 20): conv1+conv2 0.277 -> 0.271 ms and the SwiGLU GEMM 0.423 -> 0.436 ms, i.e. no gain, while the
// fraction of fast / hac scores further than 1e-3 of the score range from the fp16-storage oracle rose from 2e-4 to 7e-3 (the
// convolution outputs are the recurrence's inputs and the approximation error is systematic, not rounding noise).
__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float tanh_mufu(float x) {
    float y;
    asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float sigmoid_fast(float v) { return rcp_approx(1.0f + ex2_approx(-1.4426950408889634f * v)); }
__device__ __forceinline__ float swish_fast(float v) { return v * sigmoid_fast(v); }
__device__ __forceinline__ float tanh_fast(float v) { return fmaf(-2.0f, rcp_approx(ex2_approx(2.885390081777927f * v) + 1.0f), 1.0f); }

__device__ __forceinline__ int warp_sum_int(int v) { return __reduce_add_sync(0xffffffffu, v); }

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

__device__ __forceinline__ uint4 ldg_nc_v4(const uint4* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}

__device__ __forceinline__ float4 ldg_nc_f4(const float4* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
                 : "l"(p));
    return r;
}

}  // namespace b200
