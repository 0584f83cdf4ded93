// Shared device/host helpers for the muon_b200 C-ABI library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/muon_b200.h"

namespace mub {

// thread-local error string returned by mub_last_error()
void set_error(const char* fmt, ...);

inline int check_launch(const char* what) {
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) {
        cudaGetLastError();
        set_error("%s: %s", what, cudaGetErrorString(e));
        return -2;
    }
    return 0;
}

// number of SMs of the current device (cached per device id; read-only after first call)
int sm_count();

#define MUB_REQUIRE(cond, ...)          \
    do {                                \
        if (!(cond)) {                  \
            mub::set_error(__VA_ARGS__); \
            return -1;                  \
        }                               \
    } while (0)

constexpr int kWarp = 32;

// ---- streaming loads: CSR indices/values are read exactly once per pass, keep them out of L1
__device__ __forceinline__ int ld_stream(const int* p) {
    int v;
    asm volatile("ld.global.nc.L1::no_allocate.s32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ float ld_stream(const float* p) {
    float v;
    asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ double ld_stream(const double* p) {
    double v;
    asm volatile("ld.global.nc.L1::no_allocate.f64 %0, [%1];" : "=d"(v) : "l"(p));
    return v;
}
// same, but coherent (no .nc): for buffers that may alias an output of the same kernel
__device__ __forceinline__ float ld_stream_rw(const float* p) {
    float v;
    asm volatile("ld.global.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ double ld_stream_rw(const double* p) {
    double v;
    asm volatile("ld.global.L1::no_allocate.f64 %0, [%1];" : "=d"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ int4 ld_stream4(const int4* p) {
    int4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}
__device__ __forceinline__ int2 ld_stream2(const int2* p) {
    int2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.s32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
    return r;
}
__device__ __forceinline__ float4 ld_stream4(const float4* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
                 : "l"(p));
    return r;
}
// gather loads of the dense operand: read-only path, allowed to live in L1
__device__ __forceinline__ float4 ld_gather4(const float* p) {
    float4 r;
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
                 : "l"(p));
    return r;
}
__device__ __forceinline__ uint4 ld_gather_u4(const void* p) {
    uint4 r;
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
// streaming store
__device__ __forceinline__ void st_stream(float* p, float v) {
    asm volatile("st.global.L1::no_allocate.f32 [%0], %1;" ::"l"(p), "f"(v));
}
__device__ __forceinline__ void st_stream(double* p, double v) {
    asm volatile("st.global.L1::no_allocate.f64 [%0], %1;" ::"l"(p), "d"(v));
}

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

}  // namespace mub
