// K15 -- scOpen's bounded NMF (muon.atac.pp.scopen) on the positive pattern of the peak matrix, float64 sums.
//
//   The reference factorises the dense peaks x cells matrix X[p, c] = s_c [count(c, p) > 0].  Both products of the
//   coordinate-descent iteration are sparse gather-sums over that pattern, and every row of a factor is updated
//   independently, so nothing here is dense in cells x peaks except the imputed output, written block by block.
//
//   Kernels:
//     count_kernel    entries > 0 per CSR row (one warp per row);
//     fill_kernel     the positive entries' column indices in stored order, plus an fp32 row scale as the data of the
//                     SVD operand (one warp per row, ballot compaction);
//     spmm_kernel     C[i, :] = row_scale[i] sum_{j in pat(i)} col_scale[j] B[j, :] (one warp per row, lanes over the
//                     k <= 64 columns, the row's entries broadcast from the lane that loaded them);
//     gram_kernel     per-CTA partials of Y^T Y over a contiguous chunk of rows, summed in CTA order by reduce_kernel;
//     cd_kernel       one coordinate-descent sweep of a factor, one row per warp (sklearn's _update_cdnmf_fast with
//                     the update projected onto [0, upper]); per-CTA violation partials, summed in CTA order;
//     impute_kernel   a block of rows of clip(W H, 0, 1), one thread per output column.
//
//   The row -> warp and row -> CTA assignments depend only on the sizes and the SM count, and no sum uses float
//   atomics: two calls on the same device return the same bits.
#include <math.h>

#include "common.cuh"

namespace mub {
namespace scopen {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / kWarp;
constexpr int kTile = 32;        // rows staged per Gram tile
constexpr int kImputeRows = 16;  // output rows per impute CTA
constexpr int kMaxK = MUB_SCOPEN_MAX_COMPONENTS;

inline int row_warp_blocks(int64_t rows) {
    const int64_t want = (rows + kWarps - 1) / kWarps;
    const int64_t cap = 8 * (int64_t)sm_count();
    return (int)(want < cap ? (want < 1 ? 1 : want) : cap);
}

inline int gram_blocks(int64_t rows) {
    const int64_t want = (rows + kTile - 1) / kTile;
    const int64_t cap = 2 * (int64_t)sm_count();
    return (int)(want < cap ? (want < 1 ? 1 : want) : cap);
}

// ---- positive pattern --------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kThreads) count_kernel(const int64_t* __restrict__ indptr,
                                                         const T* __restrict__ data, int64_t rows,
                                                         int64_t* __restrict__ count) {
    const int lane = threadIdx.x % kWarp;
    const int64_t warps = (int64_t)gridDim.x * kWarps;
    for (int64_t i = (int64_t)blockIdx.x * kWarps + threadIdx.x / kWarp; i < rows; i += warps) {
        int64_t c = 0;
        for (int64_t e = indptr[i] + lane; e < indptr[i + 1]; e += kWarp) c += ld_stream(data + e) > T(0);
#pragma unroll
        for (int o = 16; o > 0; o /= 2) c += __shfl_xor_sync(0xffffffffu, c, o);
        if (lane == 0) count[i] = c;
    }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) fill_kernel(const int64_t* __restrict__ indptr,
                                                        const int32_t* __restrict__ indices,
                                                        const T* __restrict__ data, int64_t rows,
                                                        const int64_t* __restrict__ out_indptr,
                                                        const float* __restrict__ row_scale,
                                                        int32_t* __restrict__ out_indices,
                                                        float* __restrict__ out_data) {
    const int lane = threadIdx.x % kWarp;
    const int64_t warps = (int64_t)gridDim.x * kWarps;
    const unsigned below = (1u << lane) - 1u;
    for (int64_t i = (int64_t)blockIdx.x * kWarps + threadIdx.x / kWarp; i < rows; i += warps) {
        int64_t o = out_indptr[i];
        const float sc = row_scale == nullptr ? 0.0f : row_scale[i];
        for (int64_t e0 = indptr[i]; e0 < indptr[i + 1]; e0 += kWarp) {
            const int64_t e = e0 + lane;
            const bool pos = e < indptr[i + 1] && ld_stream(data + e) > T(0);
            const unsigned mask = __ballot_sync(0xffffffffu, pos);
            if (pos) {
                const int64_t at = o + __popc(mask & below);
                out_indices[at] = ld_stream(indices + e);
                if (out_data != nullptr) out_data[at] = sc;
            }
            o += __popc(mask);
        }
    }
}

// ---- pattern SpMM ------------------------------------------------------------------------------------------------
template <int J>
__global__ void __launch_bounds__(kThreads) spmm_kernel(const int64_t* __restrict__ indptr,
                                                        const int32_t* __restrict__ indices, int64_t rows,
                                                        const double* __restrict__ row_scale,
                                                        const double* __restrict__ col_scale,
                                                        const double* __restrict__ B, int k,
                                                        double* __restrict__ C) {
    const int lane = threadIdx.x % kWarp;
    const int64_t warps = (int64_t)gridDim.x * kWarps;
    for (int64_t i = (int64_t)blockIdx.x * kWarps + threadIdx.x / kWarp; i < rows; i += warps) {
        double acc[J];
#pragma unroll
        for (int q = 0; q < J; ++q) acc[q] = 0.0;
        const int64_t e1 = indptr[i + 1];
        for (int64_t e0 = indptr[i]; e0 < e1; e0 += kWarp) {
            const int64_t e = e0 + lane;
            const int j_mine = e < e1 ? ld_stream(indices + e) : 0;
            const double w_mine = e < e1 && col_scale != nullptr ? col_scale[j_mine] : 1.0;
            const int nt = (int)min((int64_t)kWarp, e1 - e0);
            for (int t = 0; t < nt; ++t) {
                const int64_t j = __shfl_sync(0xffffffffu, j_mine, t);
                const double w = __shfl_sync(0xffffffffu, w_mine, t);
                const double* b = B + j * k;
#pragma unroll
                for (int q = 0; q < J; ++q) {
                    const int c = lane + q * kWarp;
                    if (c < k) acc[q] = fma(w, b[c], acc[q]);
                }
            }
        }
        const double rs = row_scale == nullptr ? 1.0 : row_scale[i];
#pragma unroll
        for (int q = 0; q < J; ++q) {
            const int c = lane + q * kWarp;
            if (c < k) C[i * k + c] = rs * acc[q];
        }
    }
}

// ---- Gram --------------------------------------------------------------------------------------------------------
// Thread t accumulates the entries t, t + 256, ... of the row-major k x k result; J = ceil(k^2 / 256) <= 16.
template <int J>
__global__ void __launch_bounds__(kThreads) gram_kernel(const double* __restrict__ Y, int64_t rows, int k,
                                                        int64_t chunk, double* __restrict__ part) {
    __shared__ double S[kTile][kMaxK + 1];
    const int64_t r0 = (int64_t)blockIdx.x * chunk, r1 = min(rows, r0 + chunk);
    const int kk = k * k;
    double acc[J];
#pragma unroll
    for (int j = 0; j < J; ++j) acc[j] = 0.0;
    for (int64_t t0 = r0; t0 < r1; t0 += kTile) {
        const int nt = (int)min((int64_t)kTile, r1 - t0);
        __syncthreads();
        for (int e = threadIdx.x; e < nt * k; e += kThreads) S[e / k][e % k] = ld_stream(Y + t0 * k + e);
        __syncthreads();
#pragma unroll
        for (int j = 0; j < J; ++j) {
            const int o = threadIdx.x + j * kThreads;
            if (o < kk) {
                const int a = o / k, b = o % k;
                double s = acc[j];
                for (int t = 0; t < nt; ++t) s = fma(S[t][a], S[t][b], s);
                acc[j] = s;
            }
        }
    }
#pragma unroll
    for (int j = 0; j < J; ++j) {
        const int o = threadIdx.x + j * kThreads;
        if (o < kk) part[(int64_t)blockIdx.x * kk + o] = acc[j];
    }
}

__global__ void __launch_bounds__(kThreads) reduce_kernel(const double* __restrict__ part, int nblk, int64_t len,
                                                          double* __restrict__ out) {
    const int64_t e = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (e >= len) return;
    double s = 0.0;
    for (int b = 0; b < nblk; ++b) s += part[(int64_t)b * len + e];
    out[e] = s;
}

// ---- coordinate descent ------------------------------------------------------------------------------------------
// Row i of W (k <= 64: lane holds columns lane and lane + 32) is swept over the components t = 0 .. k-1 in order:
//   grad = (G + l2 I)[t, :] . w - XHt[i, t]       (warp butterfly: every lane holds the same bits)
//   pg   = w_t == 0 ? min(0, grad) : grad          (sklearn's projected gradient, summed as |pg| into the violation)
//   w_t  = min(max(w_t - grad / hess, 0), upper)   when hess = (G + l2 I)[t, t] != 0.
template <int J>
__global__ void __launch_bounds__(kThreads) cd_kernel(double* __restrict__ W, int64_t rows, int k,
                                                      const double* __restrict__ G, double l2,
                                                      const double* __restrict__ XHt, double upper,
                                                      double* __restrict__ part) {
    __shared__ double Gs[kMaxK * kMaxK];
    __shared__ double s_viol[kWarps];
    for (int e = threadIdx.x; e < k * k; e += kThreads) Gs[e] = G[e] + (e / k == e % k ? l2 : 0.0);
    __syncthreads();
    const int lane = threadIdx.x % kWarp, warp = threadIdx.x / kWarp;
    const int64_t warps = (int64_t)gridDim.x * kWarps;
    double viol = 0.0;
    for (int64_t i = (int64_t)blockIdx.x * kWarps + warp; i < rows; i += warps) {
        double w[J], x[J];
#pragma unroll
        for (int q = 0; q < J; ++q) {
            const int c = lane + q * kWarp;
            w[q] = c < k ? W[i * k + c] : 0.0;
            x[q] = c < k ? XHt[i * k + c] : 0.0;
        }
        for (int t = 0; t < k; ++t) {
            const double* g = Gs + t * k;
            double d = 0.0;
#pragma unroll
            for (int q = 0; q < J; ++q) {
                const int c = lane + q * kWarp;
                if (c < k) d = fma(g[c], w[q], d);
            }
#pragma unroll
            for (int o = 16; o > 0; o /= 2) d += __shfl_xor_sync(0xffffffffu, d, o);
            const int qt = t / kWarp, lt = t % kWarp;
            double wt = 0.0, xt = 0.0;
#pragma unroll
            for (int q = 0; q < J; ++q)
                if (q == qt) {
                    wt = __shfl_sync(0xffffffffu, w[q], lt);
                    xt = __shfl_sync(0xffffffffu, x[q], lt);
                }
            const double grad = d - xt;
            const double pg = wt == 0.0 ? fmin(0.0, grad) : grad;
            viol += fabs(pg);
            const double hess = g[t];
            if (hess != 0.0) {
                const double nw = fmin(fmax(wt - grad / hess, 0.0), upper);
#pragma unroll
                for (int q = 0; q < J; ++q)
                    if (q == qt && lane == lt) w[q] = nw;
            }
        }
#pragma unroll
        for (int q = 0; q < J; ++q) {
            const int c = lane + q * kWarp;
            if (c < k) W[i * k + c] = w[q];
        }
    }
    if (lane == 0) s_viol[warp] = viol;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int v = 0; v < kWarps; ++v) s += s_viol[v];
        part[blockIdx.x] = s;
    }
}

// ---- imputation --------------------------------------------------------------------------------------------------
// out[(p - p0) n + c] = clip(sum_r W[p, r] Ht[c, r], 0, 1) for p in [p0, p1): the CTA's rows of W in shared memory,
// Ht[c, :] in registers, r summed in order.
__global__ void __launch_bounds__(kThreads) impute_kernel(const double* __restrict__ W, int64_t p0, int64_t p1,
                                                          const double* __restrict__ Ht, int64_t n, int k,
                                                          double* __restrict__ out) {
    __shared__ double Ws[kImputeRows][kMaxK];
    const int64_t pb = p0 + (int64_t)blockIdx.y * kImputeRows;
    const int nr = (int)min((int64_t)kImputeRows, p1 - pb);
    for (int e = threadIdx.x; e < nr * k; e += kThreads) Ws[e / k][e % k] = W[(pb + e / k) * k + e % k];
    __syncthreads();
    const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (c >= n) return;
    double h[kMaxK];
#pragma unroll
    for (int r = 0; r < kMaxK; ++r) h[r] = r < k ? Ht[c * k + r] : 0.0;
    for (int p = 0; p < nr; ++p) {
        double s = 0.0;
#pragma unroll
        for (int r = 0; r < kMaxK; ++r)
            if (r < k) s = fma(Ws[p][r], h[r], s);
        out[(pb - p0 + p) * n + c] = fmin(fmax(s, 0.0), 1.0);
    }
}

// ---- host entry points -------------------------------------------------------------------------------------------
template <typename T>
int pattern_count(const int64_t* indptr, const T* data, int64_t rows, int64_t* count, cudaStream_t s) {
    MUB_REQUIRE(rows >= 0, "scopen pattern count: rows < 0");
    MUB_REQUIRE(indptr && count && (data || rows == 0), "scopen pattern count: null pointer");
    if (rows == 0) return 0;
    count_kernel<T><<<row_warp_blocks(rows), kThreads, 0, s>>>(indptr, data, rows, count);
    return check_launch("scopen count_kernel");
}

template <typename T>
int pattern_fill(const int64_t* indptr, const int32_t* indices, const T* data, int64_t rows,
                 const int64_t* out_indptr, const float* row_scale, int32_t* out_indices, float* out_data,
                 cudaStream_t s) {
    MUB_REQUIRE(rows >= 0, "scopen pattern fill: rows < 0");
    MUB_REQUIRE(indptr && out_indptr && out_indices, "scopen pattern fill: null pointer");
    MUB_REQUIRE((out_data == nullptr) == (row_scale == nullptr), "scopen pattern fill: give both or neither of "
                "row_scale and out_data");
    if (rows == 0) return 0;
    fill_kernel<T><<<row_warp_blocks(rows), kThreads, 0, s>>>(indptr, indices, data, rows, out_indptr, row_scale,
                                                               out_indices, out_data);
    return check_launch("scopen fill_kernel");
}

template <int J>
int launch_gram(const double* Y, int64_t rows, int k, double* part, int nblk, int64_t chunk, cudaStream_t s) {
    gram_kernel<J><<<nblk, kThreads, 0, s>>>(Y, rows, k, chunk, part);
    return check_launch("scopen gram_kernel");
}

}  // namespace scopen
}  // namespace mub

using namespace mub;
using namespace mub::scopen;

extern "C" {

size_t mub_scopen_workspace_bytes(int64_t rows, int32_t k) {
    if (rows < 1 || k < 1) return 0;
    const size_t gram = sizeof(double) * (size_t)k * k * (size_t)gram_blocks(rows);
    const size_t cd = sizeof(double) * (size_t)row_warp_blocks(rows);
    return gram > cd ? gram : cd;
}

int mub_scopen_pattern_count_f32(const int64_t* indptr, const float* data, int64_t rows, int64_t* count,
                                 mub_stream_t stream) {
    return pattern_count<float>(indptr, data, rows, count, (cudaStream_t)stream);
}
int mub_scopen_pattern_count_f64(const int64_t* indptr, const double* data, int64_t rows, int64_t* count,
                                 mub_stream_t stream) {
    return pattern_count<double>(indptr, data, rows, count, (cudaStream_t)stream);
}

int mub_scopen_pattern_fill_f32(const int64_t* indptr, const int32_t* indices, const float* data, int64_t rows,
                                const int64_t* out_indptr, const float* row_scale, int32_t* out_indices,
                                float* out_data, mub_stream_t stream) {
    return pattern_fill<float>(indptr, indices, data, rows, out_indptr, row_scale, out_indices, out_data,
                               (cudaStream_t)stream);
}
int mub_scopen_pattern_fill_f64(const int64_t* indptr, const int32_t* indices, const double* data, int64_t rows,
                                const int64_t* out_indptr, const float* row_scale, int32_t* out_indices,
                                float* out_data, mub_stream_t stream) {
    return pattern_fill<double>(indptr, indices, data, rows, out_indptr, row_scale, out_indices, out_data,
                                (cudaStream_t)stream);
}

int mub_scopen_spmm_f64(const int64_t* indptr, const int32_t* indices, int64_t rows, const double* row_scale,
                        const double* col_scale, const double* B, int32_t k, double* C, mub_stream_t stream) {
    MUB_REQUIRE(rows >= 0 && k >= 1 && k <= kMaxK, "scopen spmm: need rows >= 0 and 1 <= k <= %d (k=%d)", kMaxK, k);
    MUB_REQUIRE(indptr && indices && B && C, "scopen spmm: null pointer");
    if (rows == 0) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    const int nblk = row_warp_blocks(rows);
    if (k <= kWarp)
        spmm_kernel<1><<<nblk, kThreads, 0, s>>>(indptr, indices, rows, row_scale, col_scale, B, k, C);
    else
        spmm_kernel<2><<<nblk, kThreads, 0, s>>>(indptr, indices, rows, row_scale, col_scale, B, k, C);
    return check_launch("scopen spmm_kernel");
}

int mub_scopen_gram_f64(const double* Y, int64_t rows, int32_t k, void* workspace, double* G, mub_stream_t stream) {
    MUB_REQUIRE(rows >= 1 && k >= 1 && k <= kMaxK, "scopen gram: need rows >= 1 and 1 <= k <= %d (rows=%lld k=%d)",
                kMaxK, (long long)rows, k);
    MUB_REQUIRE(Y && workspace && G, "scopen gram: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    const int nblk = gram_blocks(rows);
    const int64_t chunk = (rows + nblk - 1) / nblk;
    double* part = (double*)workspace;
    const int need = (k * k + kThreads - 1) / kThreads;
    int rc;
    if (need <= 1)
        rc = launch_gram<1>(Y, rows, k, part, nblk, chunk, s);
    else if (need <= 2)
        rc = launch_gram<2>(Y, rows, k, part, nblk, chunk, s);
    else if (need <= 4)
        rc = launch_gram<4>(Y, rows, k, part, nblk, chunk, s);
    else if (need <= 8)
        rc = launch_gram<8>(Y, rows, k, part, nblk, chunk, s);
    else
        rc = launch_gram<16>(Y, rows, k, part, nblk, chunk, s);
    if (rc) return rc;
    const int64_t kk = (int64_t)k * k;
    reduce_kernel<<<(unsigned)((kk + kThreads - 1) / kThreads), kThreads, 0, s>>>(part, nblk, kk, G);
    return check_launch("scopen reduce_kernel");
}

int mub_scopen_cd_f64(double* W, int64_t rows, int32_t k, const double* G, double l2, const double* XHt, double upper,
                      void* workspace, double* violation, mub_stream_t stream) {
    MUB_REQUIRE(rows >= 1 && k >= 1 && k <= kMaxK, "scopen cd: need rows >= 1 and 1 <= k <= %d (rows=%lld k=%d)",
                kMaxK, (long long)rows, k);
    MUB_REQUIRE(W && G && XHt && workspace && violation, "scopen cd: null pointer");
    MUB_REQUIRE(upper >= 0.0, "scopen cd: upper bound %g < 0", upper);
    cudaStream_t s = (cudaStream_t)stream;
    const int nblk = row_warp_blocks(rows);
    double* part = (double*)workspace;
    if (k <= kWarp)
        cd_kernel<1><<<nblk, kThreads, 0, s>>>(W, rows, k, G, l2, XHt, upper, part);
    else
        cd_kernel<2><<<nblk, kThreads, 0, s>>>(W, rows, k, G, l2, XHt, upper, part);
    if (int rc = check_launch("scopen cd_kernel")) return rc;
    reduce_kernel<<<1, kThreads, 0, s>>>(part, nblk, 1, violation);
    return check_launch("scopen reduce_kernel");
}

int mub_scopen_impute_f64(const double* W, int64_t p0, int64_t p1, const double* Ht, int64_t n, int32_t k,
                          double* out, mub_stream_t stream) {
    MUB_REQUIRE(p0 >= 0 && p1 >= p0 && n >= 0 && k >= 1 && k <= kMaxK,
                "scopen impute: need 0 <= p0 <= p1, n >= 0 and 1 <= k <= %d (p0=%lld p1=%lld n=%lld k=%d)", kMaxK,
                (long long)p0, (long long)p1, (long long)n, k);
    MUB_REQUIRE(W && Ht && out, "scopen impute: null pointer");
    if (p1 == p0 || n == 0) return 0;
    const int64_t gy = (p1 - p0 + kImputeRows - 1) / kImputeRows;
    MUB_REQUIRE(gy <= 65535, "scopen impute: at most %d rows per call (got %lld)", 65535 * kImputeRows,
                (long long)(p1 - p0));
    const dim3 grid((unsigned)((n + kThreads - 1) / kThreads), (unsigned)gy);
    impute_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(W, p0, p1, Ht, n, k, out);
    return check_launch("scopen impute_kernel");
}

}  // extern "C"
