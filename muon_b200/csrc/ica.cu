// K14 -- the n-sized passes of FastICA (sklearn's FastICA._fit_transform as muon.tl.ica calls it), float64 sums.
//
//   Every pass splits the rows into one contiguous chunk per CTA (ica_blocks(n) CTAs, a function of n and the SM
//   count only), accumulates the chunk in a fixed order into a per-CTA partial, and reduce_kernel sums the partials
//   in CTA order.  No float atomics: two calls on the same device return the same bits.
//
//   Kernels:
//     colsum_kernel     per-CTA column sums of X (input dtype, widened), non-finite flag;
//     gram_kernel       per-CTA (X - mean)^T (X - mean): 32-row tiles centred into shared memory, a 16 x 16 thread
//                       grid with a TP x TP register tile each (the width padded to 16 TP);
//     project_kernel    X1 = Kt^T (x - mean) per row (warp = row, lane = output column), or a widening copy;
//     step_kernel       one fixed-point pass for r rows of W: per 32-row tile y = W x1 (r x 32) with g and g' in
//                       shared memory, then the r x k partial sum of g(y) x1^T in registers (J per thread);
//     sources_kernel    v = T(M x1) [/ d1, / d2, rounded to T after each division]; writes v, or accumulates the
//                       per-CTA column sums of v (mode 1) / of (v - mean)^2 (mode 2) for the ddof-0 std;
//     reduce_kernel     out[e] = (sum over CTAs in order of part[b][e]) / div; finish_std_kernel.
#include <math.h>

#include "common.cuh"

namespace mub {
namespace ica {

constexpr int kThreads = 256;
constexpr int kTile = 32;  // rows staged per tile

inline int ica_blocks(int64_t n) {
    const int64_t want = (n + kTile - 1) / kTile;
    const int64_t cap = 2 * (int64_t)sm_count();
    return (int)(want < cap ? (want < 1 ? 1 : want) : cap);
}

inline int64_t chunk_rows(int64_t n, int nblk) { return (n + nblk - 1) / nblk; }

template <typename T>
__device__ __forceinline__ T round_to(double v);
template <>
__device__ __forceinline__ float round_to<float>(double v) { return (float)v; }
template <>
__device__ __forceinline__ double round_to<double>(double v) { return v; }

// ---- column sums -------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kThreads) colsum_kernel(const T* __restrict__ X, int64_t n, int p, int64_t chunk,
                                                          double* __restrict__ part, int32_t* status) {
    __shared__ double s_half[kThreads];
    const int half = threadIdx.x / 128, c = threadIdx.x % 128;
    const int64_t r0 = (int64_t)blockIdx.x * chunk, r1 = min(n, r0 + chunk);
    double s = 0.0;
    bool bad = false;
    if (c < p)
        for (int64_t i = r0 + half; i < r1; i += 2) {
            const double v = (double)ld_stream(X + i * p + c);
            bad |= !isfinite(v);
            s += v;
        }
    s_half[threadIdx.x] = s;
    if (bad) atomicOr(status, 1);
    __syncthreads();
    if (half == 0 && c < p) part[(int64_t)blockIdx.x * p + c] = s_half[c] + s_half[128 + c];
}

// ---- centred Gram ------------------------------------------------------------------------------------------------
template <typename T, int TP>
__global__ void __launch_bounds__(kThreads) gram_kernel(const T* __restrict__ X, int64_t n, int p,
                                                        const double* __restrict__ mean, int64_t chunk,
                                                        double* __restrict__ part) {
    constexpr int P = 16 * TP;
    __shared__ double S[kTile][P];
    const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
    const int64_t r0 = (int64_t)blockIdx.x * chunk, r1 = min(n, r0 + chunk);
    double acc[TP][TP];
#pragma unroll
    for (int i = 0; i < TP; ++i)
#pragma unroll
        for (int j = 0; j < TP; ++j) acc[i][j] = 0.0;
    for (int64_t t0 = r0; t0 < r1; t0 += kTile) {
        const int nt = (int)min((int64_t)kTile, r1 - t0);
        for (int e = threadIdx.x; e < kTile * P; e += kThreads) {
            const int t = e / P, c = e % P;
            S[t][c] = t < nt && c < p ? (double)ld_stream(X + (t0 + t) * p + c) - mean[c] : 0.0;
        }
        __syncthreads();
        for (int t = 0; t < nt; ++t) {
            double a[TP], b[TP];
#pragma unroll
            for (int i = 0; i < TP; ++i) {
                a[i] = S[t][ty + 16 * i];
                b[i] = S[t][tx + 16 * i];
            }
#pragma unroll
            for (int i = 0; i < TP; ++i)
#pragma unroll
                for (int j = 0; j < TP; ++j) acc[i][j] = fma(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
    double* out = part + (int64_t)blockIdx.x * p * p;
#pragma unroll
    for (int i = 0; i < TP; ++i)
#pragma unroll
        for (int j = 0; j < TP; ++j) {
            const int a = ty + 16 * i, b = tx + 16 * j;
            if (a < p && b < p) out[a * p + b] = acc[i][j];
        }
}

// ---- projection --------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kThreads) project_kernel(const T* __restrict__ X, int64_t n, int p,
                                                           const double* __restrict__ mean,
                                                           const double* __restrict__ Kt, int k,
                                                           double* __restrict__ X1, int32_t* status) {
    extern __shared__ double S[];  // [kTile][p]
    const int lane = threadIdx.x % kWarp, warp = threadIdx.x / kWarp;
    const int64_t t0 = (int64_t)blockIdx.x * kTile;
    const int nt = (int)min((int64_t)kTile, n - t0);
    bool bad = false;
    for (int e = threadIdx.x; e < nt * p; e += kThreads) {
        const double v = (double)ld_stream(X + t0 * p + e);
        bad |= !isfinite(v);
        S[e] = Kt == nullptr ? v : v - mean[e % p];
    }
    if (bad) atomicOr(status, 1);
    __syncthreads();
    for (int t = warp; t < nt; t += kThreads / kWarp) {
        const double* x = S + t * p;
        for (int c = lane; c < k; c += kWarp) {
            double s;
            if (Kt == nullptr) {
                s = x[c];
            } else {
                s = 0.0;
                for (int a = 0; a < p; ++a) s = fma(Kt[a * k + c], x[a], s);
            }
            X1[(t0 + t) * k + c] = s;
        }
    }
}

// ---- one fixed-point pass ----------------------------------------------------------------------------------------
__device__ __forceinline__ void contrast(double y, int fun, double alpha, double& g, double& gp) {
    if (fun == MUB_ICA_LOGCOSH) {
        g = tanh(alpha * y);
        gp = alpha * (1.0 - g * g);
    } else if (fun == MUB_ICA_EXP) {
        const double e = exp(-(y * y) / 2.0);
        g = y * e;
        gp = (1.0 - y * y) * e;
    } else {
        g = y * y * y;
        gp = 3.0 * (y * y);
    }
}

template <int J>
__global__ void __launch_bounds__(kThreads) step_kernel(const double* __restrict__ X1, int64_t n, int k,
                                                        const double* __restrict__ W, int r, int fun, double alpha,
                                                        int64_t chunk, double* __restrict__ part) {
    extern __shared__ double smem[];
    const int ks = k | 1;                      // odd row stride: the y pass reads rows of Xs across lanes
    double* Ws = smem;                         // [r][k]
    double* Xs = Ws + r * k;                   // [kTile][ks]
    double* Ys = Xs + kTile * ks;              // [r][kTile] g(y)
    double* Ps = Ys + r * kTile;               // [r][kTile] g'(y)
    const int rk = r * k;
    for (int e = threadIdx.x; e < rk; e += kThreads) Ws[e] = W[e];
    const int64_t r0 = (int64_t)blockIdx.x * chunk, r1 = min(n, r0 + chunk);
    double acc[J];
#pragma unroll
    for (int j = 0; j < J; ++j) acc[j] = 0.0;
    double gsum = 0.0;
    for (int64_t t0 = r0; t0 < r1; t0 += kTile) {
        const int nt = (int)min((int64_t)kTile, r1 - t0);
        __syncthreads();
        for (int e = threadIdx.x; e < nt * k; e += kThreads) Xs[(e / k) * ks + e % k] = ld_stream(X1 + t0 * k + e);
        __syncthreads();
        for (int o = threadIdx.x; o < r * kTile; o += kThreads) {
            const int a = o / kTile, t = o % kTile;
            double g = 0.0, gp = 0.0;
            if (t < nt) {
                const double* w = Ws + a * k;
                const double* x = Xs + t * ks;
                double y = 0.0;
                for (int c = 0; c < k; ++c) y = fma(w[c], x[c], y);
                contrast(y, fun, alpha, g, gp);
            }
            Ys[o] = g;
            Ps[o] = gp;
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < J; ++j) {
            const int o = threadIdx.x + j * kThreads;
            if (o < rk) {
                const int a = o / k, c = o % k;
                const double* g = Ys + a * kTile;
                double s = 0.0;
                for (int t = 0; t < nt; ++t) s = fma(g[t], Xs[t * ks + c], s);
                acc[j] += s;
            }
        }
        if (threadIdx.x < r) {
            const double* q = Ps + threadIdx.x * kTile;
            double s = 0.0;
            for (int t = 0; t < nt; ++t) s += q[t];
            gsum += s;
        }
    }
    double* out = part + (int64_t)blockIdx.x * (rk + r);
#pragma unroll
    for (int j = 0; j < J; ++j) {
        const int o = threadIdx.x + j * kThreads;
        if (o < rk) out[o] = acc[j];
    }
    if (threadIdx.x < r) out[rk + threadIdx.x] = gsum;
}

// ---- sources -----------------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ double source_value(const double* __restrict__ Mt, int k, const double* x, int c,
                                               const double* __restrict__ d1, const double* __restrict__ d2) {
    double s = 0.0;
    for (int a = 0; a < k; ++a) s = fma(Mt[a * k + c], x[a], s);
    double v = (double)round_to<T>(s);
    if (d1 != nullptr) v = (double)round_to<T>(v / d1[c]);
    if (d2 != nullptr) v = (double)round_to<T>(v / d2[c]);
    return v;
}

// mode 0: out = v;  mode 1: part[b][c] = sum of v over the CTA's rows;  mode 2: the same for (v - mean[c])^2
template <typename T>
__global__ void __launch_bounds__(kThreads) sources_kernel(const double* __restrict__ X1, int64_t n, int k,
                                                           const double* __restrict__ Mt,
                                                           const double* __restrict__ d1,
                                                           const double* __restrict__ d2, int mode,
                                                           const double* __restrict__ mean, int64_t chunk,
                                                           T* __restrict__ out, double* __restrict__ part) {
    extern __shared__ double S[];  // [kTile][k], then [kThreads / kWarp][k] warp sums
    const int lane = threadIdx.x % kWarp, warp = threadIdx.x / kWarp;
    constexpr int kWarps = kThreads / kWarp;
    constexpr int kCols = MUB_ICA_MAX_DIM / kWarp;
    double* Wsum = S + kTile * k;
    const int64_t r0 = (int64_t)blockIdx.x * chunk, r1 = min(n, r0 + chunk);
    double acc[kCols];
#pragma unroll
    for (int q = 0; q < kCols; ++q) acc[q] = 0.0;
    for (int64_t t0 = r0; t0 < r1; t0 += kTile) {
        const int nt = (int)min((int64_t)kTile, r1 - t0);
        __syncthreads();
        for (int e = threadIdx.x; e < nt * k; e += kThreads) S[e] = ld_stream(X1 + t0 * k + e);
        __syncthreads();
        for (int t = warp; t < nt; t += kWarps) {
#pragma unroll
            for (int q = 0; q < kCols; ++q) {
                const int c = lane + q * kWarp;
                if (c < k) {
                    const double v = source_value<T>(Mt, k, S + t * k, c, d1, d2);
                    if (mode == 0) {
                        out[(t0 + t) * k + c] = round_to<T>(v);
                    } else if (mode == 1) {
                        acc[q] += v;
                    } else {
                        const double dv = v - mean[c];
                        acc[q] = fma(dv, dv, acc[q]);
                    }
                }
            }
        }
    }
    if (mode == 0) return;
    __syncthreads();
#pragma unroll
    for (int q = 0; q < kCols; ++q) {
        const int c = lane + q * kWarp;
        if (c < k) Wsum[warp * k + c] = acc[q];
    }
    __syncthreads();
    for (int c = threadIdx.x; c < k; c += kThreads) {
        double s = 0.0;
        for (int w = 0; w < kWarps; ++w) s += Wsum[w * k + c];
        part[(int64_t)blockIdx.x * k + c] = s;
    }
}

// ---- reductions --------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) reduce_kernel(const double* __restrict__ part, int nblk, int64_t len,
                                                          double div, double* __restrict__ out) {
    const int64_t e = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (e >= len) return;
    double s = 0.0;
    for (int b = 0; b < nblk; ++b) s += part[(int64_t)b * len + e];
    out[e] = s / div;
}

__global__ void finish_std_kernel(double* stats, int k) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < k) stats[k + c] = sqrt(stats[k + c]);
}

inline int reduce(const double* part, int nblk, int64_t len, double div, double* out, cudaStream_t s) {
    reduce_kernel<<<(unsigned)((len + kThreads - 1) / kThreads), kThreads, 0, s>>>(part, nblk, len, div, out);
    return check_launch("ica reduce_kernel");
}

inline size_t step_smem(int k, int r) {
    return sizeof(double) * ((size_t)r * k + (size_t)kTile * (k | 1) + 2 * (size_t)r * kTile);
}

// ---- host entry points -------------------------------------------------------------------------------------------
template <typename T>
int moments(const T* X, int64_t n, int32_t p, void* ws, double* mean, double* gram, int32_t* status,
            cudaStream_t s) {
    MUB_REQUIRE(n >= 1 && p >= 1 && p <= MUB_ICA_MAX_DIM, "ica moments: need n >= 1 and 1 <= p <= %d (n=%lld p=%d)",
                MUB_ICA_MAX_DIM, (long long)n, p);
    MUB_REQUIRE(X && ws && mean && gram && status, "ica moments: null pointer");
    const int nblk = ica_blocks(n);
    const int64_t chunk = chunk_rows(n, nblk);
    double* part = (double*)ws;
    colsum_kernel<T><<<nblk, kThreads, 0, s>>>(X, n, p, chunk, part, status);
    if (int rc = check_launch("ica colsum_kernel")) return rc;
    if (int rc = reduce(part, nblk, p, (double)n, mean, s)) return rc;
    if (p <= 16)
        gram_kernel<T, 1><<<nblk, kThreads, 0, s>>>(X, n, p, mean, chunk, part);
    else if (p <= 32)
        gram_kernel<T, 2><<<nblk, kThreads, 0, s>>>(X, n, p, mean, chunk, part);
    else if (p <= 64)
        gram_kernel<T, 4><<<nblk, kThreads, 0, s>>>(X, n, p, mean, chunk, part);
    else
        gram_kernel<T, 8><<<nblk, kThreads, 0, s>>>(X, n, p, mean, chunk, part);
    if (int rc = check_launch("ica gram_kernel")) return rc;
    return reduce(part, nblk, (int64_t)p * p, 1.0, gram, s);
}

template <typename T>
int project(const T* X, int64_t n, int32_t p, const double* mean, const double* Kt, int32_t k, double* X1,
            int32_t* status, cudaStream_t s) {
    MUB_REQUIRE(n >= 1 && p >= 1 && p <= MUB_ICA_MAX_DIM && k >= 1 && k <= p,
                "ica project: need n >= 1, 1 <= k <= p <= %d (n=%lld p=%d k=%d)", MUB_ICA_MAX_DIM, (long long)n, p, k);
    MUB_REQUIRE(X && X1 && status, "ica project: null pointer");
    MUB_REQUIRE(Kt == nullptr ? k == p : mean != nullptr, "ica project: a copy needs k == p, a projection a mean");
    const size_t smem = sizeof(double) * kTile * p;
    project_kernel<T><<<(unsigned)((n + kTile - 1) / kTile), kThreads, smem, s>>>(X, n, p, mean, Kt, k, X1, status);
    return check_launch("ica project_kernel");
}

template <int J>
int launch_step(const double* X1, int64_t n, int k, const double* W, int r, int fun, double alpha, int nblk,
                int64_t chunk, double* part, cudaStream_t s) {
    const size_t smem = step_smem(k, r);
    cudaError_t e = cudaFuncSetAttribute(step_kernel<J>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) {
        set_error("ica step: shared memory attribute: %s", cudaGetErrorString(e));
        return -2;
    }
    step_kernel<J><<<nblk, kThreads, smem, s>>>(X1, n, k, W, r, fun, alpha, chunk, part);
    return check_launch("ica step_kernel");
}

template <typename T>
int sources(const double* X1, int64_t n, int32_t k, const double* Mt, const double* d1, const double* d2, T* out,
            void* ws, double* stats, cudaStream_t s) {
    MUB_REQUIRE(n >= 1 && k >= 1 && k <= MUB_ICA_MAX_DIM, "ica sources: need n >= 1 and 1 <= k <= %d (n=%lld k=%d)",
                MUB_ICA_MAX_DIM, (long long)n, k);
    MUB_REQUIRE(X1 && Mt, "ica sources: null pointer");
    MUB_REQUIRE((stats != nullptr) != (out != nullptr), "ica sources: give exactly one of out and stats");
    MUB_REQUIRE(stats == nullptr || ws != nullptr, "ica sources: stats need the workspace");
    const size_t smem = sizeof(double) * ((size_t)kTile * k + (size_t)(kThreads / kWarp) * k);
    if (out != nullptr) {
        const int nblk = (int)((n + kTile - 1) / kTile);
        sources_kernel<T><<<nblk, kThreads, smem, s>>>(X1, n, k, Mt, d1, d2, 0, nullptr, kTile, out, nullptr);
        return check_launch("ica sources_kernel");
    }
    const int nblk = ica_blocks(n);
    const int64_t chunk = chunk_rows(n, nblk);
    double* part = (double*)ws;
    sources_kernel<T><<<nblk, kThreads, smem, s>>>(X1, n, k, Mt, d1, d2, 1, nullptr, chunk, nullptr, part);
    if (int rc = check_launch("ica sources_kernel")) return rc;
    if (int rc = reduce(part, nblk, k, (double)n, stats, s)) return rc;
    sources_kernel<T><<<nblk, kThreads, smem, s>>>(X1, n, k, Mt, d1, d2, 2, stats, chunk, nullptr, part);
    if (int rc = check_launch("ica sources_kernel")) return rc;
    if (int rc = reduce(part, nblk, k, (double)n, stats + k, s)) return rc;
    finish_std_kernel<<<(k + 127) / 128, 128, 0, s>>>(stats, k);
    return check_launch("ica finish_std_kernel");
}

}  // namespace ica
}  // namespace mub

using namespace mub::ica;

extern "C" {

size_t mub_ica_workspace_bytes(int64_t n, int32_t p, int32_t k) {
    if (n < 1 || p < 1 || k < 1) return 0;
    const size_t per = (size_t)p * p + p > (size_t)k * k + k ? (size_t)p * p + p : (size_t)k * k + k;
    return sizeof(double) * per * (size_t)ica_blocks(n);
}

int mub_ica_moments_f32(const float* X, int64_t n, int32_t p, void* workspace, double* mean, double* gram,
                        int32_t* status, mub_stream_t stream) {
    return moments<float>(X, n, p, workspace, mean, gram, status, (cudaStream_t)stream);
}
int mub_ica_moments_f64(const double* X, int64_t n, int32_t p, void* workspace, double* mean, double* gram,
                        int32_t* status, mub_stream_t stream) {
    return moments<double>(X, n, p, workspace, mean, gram, status, (cudaStream_t)stream);
}

int mub_ica_project_f32(const float* X, int64_t n, int32_t p, const double* mean, const double* Kt, int32_t k,
                        double* X1, int32_t* status, mub_stream_t stream) {
    return project<float>(X, n, p, mean, Kt, k, X1, status, (cudaStream_t)stream);
}
int mub_ica_project_f64(const double* X, int64_t n, int32_t p, const double* mean, const double* Kt, int32_t k,
                        double* X1, int32_t* status, mub_stream_t stream) {
    return project<double>(X, n, p, mean, Kt, k, X1, status, (cudaStream_t)stream);
}

int mub_ica_step_f64(const double* X1, int64_t n, int32_t k, const double* W, int32_t r, int32_t fun, double alpha,
                     void* workspace, double* out, mub_stream_t stream) {
    MUB_REQUIRE(n >= 1 && k >= 1 && k <= MUB_ICA_MAX_DIM && r >= 1 && r <= k,
                "ica step: need n >= 1, 1 <= r <= k <= %d (n=%lld k=%d r=%d)", MUB_ICA_MAX_DIM, (long long)n, k, r);
    MUB_REQUIRE(fun == MUB_ICA_LOGCOSH || fun == MUB_ICA_EXP || fun == MUB_ICA_CUBE, "ica step: unknown fun %d", fun);
    MUB_REQUIRE(X1 && W && workspace && out, "ica step: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    const int nblk = ica_blocks(n);
    const int64_t chunk = chunk_rows(n, nblk);
    double* part = (double*)workspace;
    const int need = (r * k + kThreads - 1) / kThreads;
    int rc;
    if (need <= 1)
        rc = launch_step<1>(X1, n, k, W, r, fun, alpha, nblk, chunk, part, s);
    else if (need <= 2)
        rc = launch_step<2>(X1, n, k, W, r, fun, alpha, nblk, chunk, part, s);
    else if (need <= 4)
        rc = launch_step<4>(X1, n, k, W, r, fun, alpha, nblk, chunk, part, s);
    else if (need <= 8)
        rc = launch_step<8>(X1, n, k, W, r, fun, alpha, nblk, chunk, part, s);
    else if (need <= 16)
        rc = launch_step<16>(X1, n, k, W, r, fun, alpha, nblk, chunk, part, s);
    else if (need <= 32)
        rc = launch_step<32>(X1, n, k, W, r, fun, alpha, nblk, chunk, part, s);
    else
        rc = launch_step<64>(X1, n, k, W, r, fun, alpha, nblk, chunk, part, s);
    if (rc) return rc;
    return reduce(part, nblk, (int64_t)r * k + r, 1.0, out, s);
}

int mub_ica_sources_f32(const double* X1, int64_t n, int32_t k, const double* Mt, const double* d1, const double* d2,
                        float* out, void* workspace, double* stats, mub_stream_t stream) {
    return sources<float>(X1, n, k, Mt, d1, d2, out, workspace, stats, (cudaStream_t)stream);
}
int mub_ica_sources_f64(const double* X1, int64_t n, int32_t k, const double* Mt, const double* d1, const double* d2,
                        double* out, void* workspace, double* stats, mub_stream_t stream) {
    return sources<double>(X1, n, k, Mt, d1, d2, out, workspace, stats, (cudaStream_t)stream);
}

}  // extern "C"
