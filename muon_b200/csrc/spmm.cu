// K2/K3 -- CSR x dense SpMM  C[n x P] (+)= A[n x d] * B[d x P]  for sm_90a, P in {32,64,128}.
//
// Replaces the per-Lanczos-step csr_matvec/csc_matvec pair that ARPACK drives inside
// scipy.sparse.linalg.svds (scipy _svds.py:428-460, called at muon/_atac/tools.py:53) by a
// blocked operator application on P vectors at once, and mofapy2's dense Y^T Z / Y W
// contractions (muon/_core/tools.py:583-585).  A^T * Y uses the same kernel on the CSR of
// A^T (transpose.cu).
//
// v1 "row-warp" kernel: a warp owns a row.  Lane layout: P/4 lanes cover one dense row as
// float4 (16 B per lane, 4P bytes per non-zero, fully coalesced), so a warp consumes
// G = 128/P non-zeros per gather instruction.  Column indices and values are streamed in
// coalesced 128 B segments (32 per warp load, L1::no_allocate) and broadcast by shuffle;
// 32/G independent float4 gathers are in flight per lane.  fp32 FMA accumulation in
// registers, one float4 store per lane group at the end of the row.
//
// Traffic model (DESIGN.md): HBM streams 8 B/nnz (+ dense operands once); every non-zero
// additionally pulls 4P bytes of B through L2->L1, which is the practical limiter at P>=32.
#include <cuda_fp16.h>

#include "common.cuh"

namespace mub {

constexpr int kSpmmThreads = 256;
constexpr int kSpmmWarps = kSpmmThreads / kWarp;

// PAIRS: the matrix stores interleaved (column, value) pairs (int2; transposed panels) instead of two arrays
template <bool PAIRS>
__device__ __forceinline__ void load_entry(const int32_t* __restrict__ indices, const float* __restrict__ data,
                                           int64_t k, int& c, float& v) {
    if constexpr (PAIRS) {
        const int2 e = ld_stream2(reinterpret_cast<const int2*>(indices) + k);
        c = e.x;
        v = __int_as_float(e.y);
    } else {
        c = ld_stream(indices + k);
        v = ld_stream(data + k);
    }
}

template <int P, bool PAIRS>
__device__ __forceinline__ void spmm_row(const int32_t* __restrict__ indices, const float* __restrict__ data,
                                         int64_t start, int64_t end, const float* __restrict__ B,
                                         float* __restrict__ C_row, int accumulate, int lane) {
    constexpr int LPN = P / 4;    // lanes per non-zero
    constexpr int G = 32 / LPN;   // non-zeros per warp-wide gather
    constexpr int STEPS = 32 / G; // gathers per 32-nnz segment
    const int sub = lane % LPN, grp = lane / LPN;
    const float* Bl = B + sub * 4;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    int64_t base = start;
    // full 32-nnz segments: all STEPS gathers issued back to back; the next segment's (index, value) entries are
    // requested from HBM before the gathers of the current one (see spmm_row_h)
    int c_next = 0;
    float v_next = 0.f;
    bool more = base + 32 <= end;
    if (more) load_entry<PAIRS>(indices, data, base + lane, c_next, v_next);
    for (; more; base += 32) {
        const int c = c_next;
        const float v = v_next;
        more = base + 64 <= end;
        if (more) load_entry<PAIRS>(indices, data, base + 32 + lane, c_next, v_next);
        constexpr int BATCH = STEPS < 16 ? STEPS : 16;  // gathers in flight per lane
#pragma unroll
        for (int t0 = 0; t0 < STEPS; t0 += BATCH) {
            float4 b[BATCH];
            float vv[BATCH];
#pragma unroll
            for (int t = 0; t < BATCH; ++t) {
                const int cc = __shfl_sync(0xffffffffu, c, (t0 + t) * G + grp);
                vv[t] = __shfl_sync(0xffffffffu, v, (t0 + t) * G + grp);
                b[t] = ld_gather4(Bl + (size_t)cc * P);
            }
#pragma unroll
            for (int t = 0; t < BATCH; ++t) {
                acc.x = fmaf(vv[t], b[t].x, acc.x);
                acc.y = fmaf(vv[t], b[t].y, acc.y);
                acc.z = fmaf(vv[t], b[t].z, acc.z);
                acc.w = fmaf(vv[t], b[t].w, acc.w);
            }
        }
    }
    if (base < end) {  // tail segment (warp-uniform trip count)
        const int cnt = (int)(end - base);
        const bool ok = lane < cnt;
        int c = 0;
        float v = 0.f;
        if (ok) load_entry<PAIRS>(indices, data, base + lane, c, v);
        const int steps = (cnt + G - 1) / G;
        for (int t = 0; t < steps; ++t) {
            const int src = t * G + grp;
            const int cc = __shfl_sync(0xffffffffu, c, src);
            const float vt = __shfl_sync(0xffffffffu, v, src);
            if (src < cnt) {
                const float4 bt = ld_gather4(Bl + (size_t)cc * P);
                acc.x = fmaf(vt, bt.x, acc.x);
                acc.y = fmaf(vt, bt.y, acc.y);
                acc.z = fmaf(vt, bt.z, acc.z);
                acc.w = fmaf(vt, bt.w, acc.w);
            }
        }
    }
    // combine the G lane groups (fixed butterfly order: deterministic)
#pragma unroll
    for (int off = LPN; off < 32; off <<= 1) {
        acc.x += __shfl_xor_sync(0xffffffffu, acc.x, off);
        acc.y += __shfl_xor_sync(0xffffffffu, acc.y, off);
        acc.z += __shfl_xor_sync(0xffffffffu, acc.z, off);
        acc.w += __shfl_xor_sync(0xffffffffu, acc.w, off);
    }
    if (grp == 0) {
        float4* dst = reinterpret_cast<float4*>(C_row + sub * 4);
        if (accumulate) {
            const float4 o = *dst;
            acc.x += o.x; acc.y += o.y; acc.z += o.z; acc.w += o.w;
        }
        *dst = acc;
    }
}

template <int P, bool PAIRS>
__global__ void __launch_bounds__(kSpmmThreads)
spmm_csr_rowwarp_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                        const float* __restrict__ data, int64_t n_rows, const float* __restrict__ B,
                        float* __restrict__ C, int accumulate, unsigned long long* row_counter) {
    const int lane = threadIdx.x & 31;
    if (row_counter == nullptr) {
        const int64_t warp = (int64_t)blockIdx.x * kSpmmWarps + (threadIdx.x >> 5);
        const int64_t n_warps = (int64_t)gridDim.x * kSpmmWarps;
        for (int64_t row = warp; row < n_rows; row += n_warps) {
            const int64_t s = __ldg(indptr + row), e = __ldg(indptr + row + 1);
            spmm_row<P, PAIRS>(indices, data, s, e, B, C + (size_t)row * P, accumulate, lane);
        }
    } else {
        // dynamic scheduling: each warp claims the next unprocessed row (rows are issued in
        // order, so long rows of a skewed matrix cannot pile up on one warp's static list)
        for (;;) {
            unsigned long long row = 0;
            if (lane == 0) row = atomicAdd(row_counter, 1ull);
            row = __shfl_sync(0xffffffffu, row, 0);
            if ((int64_t)row >= n_rows) break;
            const int64_t s = __ldg(indptr + row), e = __ldg(indptr + row + 1);
            spmm_row<P, PAIRS>(indices, data, s, e, B, C + (size_t)row * P, accumulate, lane);
        }
    }
}

// ---- half-precision dense operand -------------------------------------------------------------------
// Same row-warp product with B stored as IEEE half (row = 2P bytes): every non-zero gathers half the bytes
// through L2 -> L1 -> registers, which is what bounds the fp32 kernel (DESIGN.md section 4).  Products and
// sums are fp32 (half -> float conversion is exact), only the operand is rounded (2^-11 relative).  Used
// by the early block-Lanczos steps of the LSI driver (_lsi.py), whose accuracy need not exceed 1e-3;
// the final steps run the fp32 kernel above.  Lane layout: P/8 lanes cover one row of B (16 B = 8 halves
// per lane), a warp consumes G = 256/P non-zeros per gather instruction.  out_scale undoes the power-of-
// two scaling the caller applied before rounding (mub_f32_to_f16_scaled).
template <int P, bool PAIRS>
__device__ __forceinline__ void spmm_row_h(const int32_t* __restrict__ indices, const float* __restrict__ data,
                                           int64_t start, int64_t end, const __half* __restrict__ B,
                                           float* __restrict__ C_row, int accumulate, float out_scale, int lane) {
    constexpr int LPN = P / 8;      // lanes per non-zero
    constexpr int G = 32 / LPN;     // non-zeros per warp-wide gather
    constexpr int STEPS = 32 / G;   // gathers per 32-nnz segment
    const int sub = lane % LPN, grp = lane / LPN;
    const __half* Bl = B + sub * 8;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    auto fma8 = [&](float v, const uint4& q) {
        const unsigned w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
            acc[2 * i] = fmaf(v, f.x, acc[2 * i]);
            acc[2 * i + 1] = fmaf(v, f.y, acc[2 * i + 1]);
        }
    };
    int64_t base = start;
    // the (index, value) stream comes from HBM (~600 ns), the gathers from L2 (~130 ns): fetch the NEXT segment's
    // entries before gathering for the current one, so a warp never waits for both latencies in sequence
    int c_next = 0;
    float v_next = 0.f;
    bool more = base + 32 <= end;
    if (more) load_entry<PAIRS>(indices, data, base + lane, c_next, v_next);
    while (more) {
        const int c = c_next;
        const float v = v_next;
        more = base + 64 <= end;
        if (more) load_entry<PAIRS>(indices, data, base + 32 + lane, c_next, v_next);
        uint4 b[STEPS];
        float vv[STEPS];
#pragma unroll
        for (int t = 0; t < STEPS; ++t) {
            const int cc = __shfl_sync(0xffffffffu, c, t * G + grp);
            vv[t] = __shfl_sync(0xffffffffu, v, t * G + grp);
            b[t] = ld_gather_u4(Bl + (size_t)cc * P);
        }
#pragma unroll
        for (int t = 0; t < STEPS; ++t) fma8(vv[t], b[t]);
        base += 32;
    }
    if (base < end) {
        const int cnt = (int)(end - base);
        const bool ok = lane < cnt;
        int c = 0;
        float v = 0.f;
        if (ok) load_entry<PAIRS>(indices, data, base + lane, c, v);
        const int steps = (cnt + G - 1) / G;
        for (int t = 0; t < steps; ++t) {
            const int src = t * G + grp;
            const int cc = __shfl_sync(0xffffffffu, c, src & 31);
            const float vt = __shfl_sync(0xffffffffu, v, src & 31);
            if (src < cnt) fma8(vt, ld_gather_u4(Bl + (size_t)cc * P));
        }
    }
#pragma unroll
    for (int off = LPN; off < 32; off <<= 1) {
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], off);
    }
    if (grp == 0) {
        float4* dst = reinterpret_cast<float4*>(C_row + sub * 8);
        float4 lo = make_float4(acc[0] * out_scale, acc[1] * out_scale, acc[2] * out_scale, acc[3] * out_scale);
        float4 hi = make_float4(acc[4] * out_scale, acc[5] * out_scale, acc[6] * out_scale, acc[7] * out_scale);
        if (accumulate) {
            const float4 o0 = dst[0], o1 = dst[1];
            lo.x += o0.x; lo.y += o0.y; lo.z += o0.z; lo.w += o0.w;
            hi.x += o1.x; hi.y += o1.y; hi.z += o1.z; hi.w += o1.w;
        }
        dst[0] = lo;
        dst[1] = hi;
    }
}

template <int P, bool PAIRS>
__global__ void __launch_bounds__(kSpmmThreads)
spmm_csr_rowwarp_h_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                          const float* __restrict__ data, int64_t n_rows, const __half* __restrict__ B,
                          float* __restrict__ C, int accumulate, float out_scale, unsigned long long* row_counter) {
    const int lane = threadIdx.x & 31;
    if (row_counter == nullptr) {
        const int64_t warp = (int64_t)blockIdx.x * kSpmmWarps + (threadIdx.x >> 5);
        const int64_t n_warps = (int64_t)gridDim.x * kSpmmWarps;
        for (int64_t row = warp; row < n_rows; row += n_warps) {
            const int64_t s = __ldg(indptr + row), e = __ldg(indptr + row + 1);
            spmm_row_h<P, PAIRS>(indices, data, s, e, B, C + (size_t)row * P, accumulate, out_scale, lane);
        }
    } else {
        for (;;) {
            unsigned long long row = 0;
            if (lane == 0) row = atomicAdd(row_counter, 1ull);
            row = __shfl_sync(0xffffffffu, row, 0);
            if ((int64_t)row >= n_rows) break;
            const int64_t s = __ldg(indptr + row), e = __ldg(indptr + row + 1);
            spmm_row_h<P, PAIRS>(indices, data, s, e, B, C + (size_t)row * P, accumulate, out_scale, lane);
        }
    }
}

template <int P, bool PAIRS>
static int launch_spmm_h(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_rows,
                         const __half* B, float* C, int accumulate, float out_scale, unsigned long long* row_counter,
                         cudaStream_t stream) {
    int64_t want = (n_rows + kSpmmWarps - 1) / kSpmmWarps;
    int64_t cap = (int64_t)sm_count() * 8;
    int grid = (int)(want < cap ? want : cap);
    if (grid < 1) grid = 1;
    spmm_csr_rowwarp_h_kernel<P, PAIRS><<<grid, kSpmmThreads, 0, stream>>>(indptr, indices, data, n_rows, B, C,
                                                                     accumulate, out_scale, row_counter);
    return check_launch("spmm_csr_h16");
}

// dst[i] = half(src[i] * scale): the rounding step in front of the half-operand products
__global__ void __launch_bounds__(256)
f32_to_f16_scaled_kernel(const float4* __restrict__ src, int64_t n4, float scale, uint2* __restrict__ dst) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        const float4 v = src[i];
        const __half2 a = __floats2half2_rn(v.x * scale, v.y * scale);
        const __half2 b = __floats2half2_rn(v.z * scale, v.w * scale);
        uint2 o;
        o.x = *reinterpret_cast<const unsigned*>(&a);
        o.y = *reinterpret_cast<const unsigned*>(&b);
        dst[i] = o;
    }
}

template <int P, bool PAIRS>
static int launch_spmm(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_rows,
                       const float* B, float* C, int accumulate, unsigned long long* row_counter,
                       cudaStream_t stream) {
    int64_t want = (n_rows + kSpmmWarps - 1) / kSpmmWarps;
    int64_t cap = (int64_t)sm_count() * 8;  // 2048 threads / SM
    int grid = (int)(want < cap ? want : cap);
    if (grid < 1) grid = 1;
    spmm_csr_rowwarp_kernel<P, PAIRS><<<grid, kSpmmThreads, 0, stream>>>(indptr, indices, data, n_rows, B, C,
                                                                   accumulate, row_counter);
    return check_launch("spmm_csr");
}

}  // namespace mub

extern "C" int mub_spmm_csr_f32(const int64_t* indptr, const int32_t* indices, const float* data,
                                int64_t n_rows, int64_t n_cols, const float* B, int32_t ld, float* C,
                                int32_t accumulate, unsigned long long* row_counter, mub_stream_t stream) {
    MUB_REQUIRE(n_rows >= 0 && n_cols >= 0, "spmm_csr: negative shape");
    MUB_REQUIRE(ld == 32 || ld == 64 || ld == 128, "spmm_csr: ld must be 32, 64 or 128 (got %d)", ld);
    if (n_rows == 0) return 0;
    MUB_REQUIRE(indptr && B && C, "spmm_csr: null pointer");
    MUB_REQUIRE((((uintptr_t)B | (uintptr_t)C) & 15) == 0, "spmm_csr: B and C must be 16-byte aligned");
    cudaStream_t s = (cudaStream_t)stream;
    switch (ld) {
        case 32: return mub::launch_spmm<32, false>(indptr, indices, data, n_rows, B, C, accumulate, row_counter, s);
        case 64: return mub::launch_spmm<64, false>(indptr, indices, data, n_rows, B, C, accumulate, row_counter, s);
        default: return mub::launch_spmm<128, false>(indptr, indices, data, n_rows, B, C, accumulate, row_counter, s);
    }
}

extern "C" int mub_spmm_csrp_f32(const int64_t* indptr, const int32_t* pairs, int64_t n_rows, int64_t n_cols,
                                 const float* B, int32_t ld, float* C, int32_t accumulate,
                                 unsigned long long* row_counter, mub_stream_t stream) {
    MUB_REQUIRE(n_rows >= 0 && n_cols >= 0, "spmm_csrp: negative shape");
    MUB_REQUIRE(ld == 32 || ld == 64 || ld == 128, "spmm_csrp: ld must be 32, 64 or 128 (got %d)", ld);
    if (n_rows == 0) return 0;
    MUB_REQUIRE(indptr && B && C, "spmm_csrp: null pointer");
    MUB_REQUIRE((((uintptr_t)B | (uintptr_t)C) & 15) == 0 && ((uintptr_t)pairs & 7) == 0, "spmm_csrp: misaligned operand");
    cudaStream_t s = (cudaStream_t)stream;
    switch (ld) {
        case 32: return mub::launch_spmm<32, true>(indptr, pairs, nullptr, n_rows, B, C, accumulate, row_counter, s);
        case 64: return mub::launch_spmm<64, true>(indptr, pairs, nullptr, n_rows, B, C, accumulate, row_counter, s);
        default: return mub::launch_spmm<128, true>(indptr, pairs, nullptr, n_rows, B, C, accumulate, row_counter, s);
    }
}

// ---- half-precision dense operand (see spmm_row_h) ---------------------------------------------------
extern "C" int mub_f32_to_f16_scaled(const float* src, int64_t n, float scale, void* dst, mub_stream_t stream) {
    MUB_REQUIRE(n >= 0 && (n % 4) == 0, "f32_to_f16_scaled: n must be a non-negative multiple of 4");
    if (n == 0) return 0;
    MUB_REQUIRE(src && dst && (((uintptr_t)src & 15) == 0) && (((uintptr_t)dst & 7) == 0), "f32_to_f16_scaled: misaligned operand");
    int64_t want = (n / 4 + 255) / 256, cap = (int64_t)mub::sm_count() * 8;
    int grid = (int)(want < cap ? want : cap);
    mub::f32_to_f16_scaled_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const float4*)src, n / 4, scale, (uint2*)dst);
    return mub::check_launch("f32_to_f16_scaled");
}

extern "C" int mub_spmm_csr_h16(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_rows,
                                int64_t n_cols, const void* B_half, int32_t ld, float* C, int32_t accumulate,
                                float out_scale, unsigned long long* row_counter, mub_stream_t stream) {
    MUB_REQUIRE(n_rows >= 0 && n_cols >= 0, "spmm_csr_h16: negative shape");
    MUB_REQUIRE(ld == 32 || ld == 64 || ld == 128, "spmm_csr_h16: ld must be 32, 64 or 128 (got %d)", ld);
    if (n_rows == 0) return 0;
    MUB_REQUIRE(indptr && B_half && C, "spmm_csr_h16: null pointer");
    MUB_REQUIRE((((uintptr_t)B_half | (uintptr_t)C) & 15) == 0, "spmm_csr_h16: B and C must be 16-byte aligned");
    cudaStream_t s = (cudaStream_t)stream;
    const __half* B = (const __half*)B_half;
    switch (ld) {
        case 32: return mub::launch_spmm_h<32, false>(indptr, indices, data, n_rows, B, C, accumulate, out_scale, row_counter, s);
        case 64: return mub::launch_spmm_h<64, false>(indptr, indices, data, n_rows, B, C, accumulate, out_scale, row_counter, s);
        default: return mub::launch_spmm_h<128, false>(indptr, indices, data, n_rows, B, C, accumulate, out_scale, row_counter, s);
    }
}

extern "C" int mub_spmm_csrp_h16(const int64_t* indptr, const int32_t* pairs, int64_t n_rows, int64_t n_cols,
                                 const void* B_half, int32_t ld, float* C, int32_t accumulate, float out_scale,
                                 unsigned long long* row_counter, mub_stream_t stream) {
    MUB_REQUIRE(n_rows >= 0 && n_cols >= 0, "spmm_csrp_h16: negative shape");
    MUB_REQUIRE(ld == 32 || ld == 64 || ld == 128, "spmm_csrp_h16: ld must be 32, 64 or 128 (got %d)", ld);
    if (n_rows == 0) return 0;
    MUB_REQUIRE(indptr && B_half && C, "spmm_csrp_h16: null pointer");
    MUB_REQUIRE((((uintptr_t)B_half | (uintptr_t)C) & 15) == 0 && ((uintptr_t)pairs & 7) == 0, "spmm_csrp_h16: misaligned operand");
    cudaStream_t s = (cudaStream_t)stream;
    const __half* B = (const __half*)B_half;
    switch (ld) {
        case 32: return mub::launch_spmm_h<32, true>(indptr, pairs, nullptr, n_rows, B, C, accumulate, out_scale, row_counter, s);
        case 64: return mub::launch_spmm_h<64, true>(indptr, pairs, nullptr, n_rows, B, C, accumulate, out_scale, row_counter, s);
        default: return mub::launch_spmm_h<128, true>(indptr, pairs, nullptr, n_rows, B, C, accumulate, out_scale, row_counter, s);
    }
}
