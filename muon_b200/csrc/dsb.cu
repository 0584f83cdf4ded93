// K8 -- DSB normalisation of CITE-seq protein counts (reference arithmetic: muon/_prot/preproc.py:161-218).
//
//   moments : two passes over the empty droplets (CSR or dense): per-protein fp64 sums of d = log(x+pc) - log(pc),
//             then of (d - mean d)^2 (a one-pass sum of d^2 loses ~1e-12 of the std to cancellation).  Shifting
//             by the value of an implicit zero means only stored entries are read.  Each block owns a fixed row
//             range and writes its partial sums; a second kernel adds the partials in block order, so the
//             result is bit-identical from run to run (no float atomics).
//   fit     : one warp per cell.  The warp scales its row (preproc.py:161-177, rounded to the output dtype like
//             the reference), writes it, and fits the two 2-component Gaussian mixtures of preproc.py:183-198
//             (sklearn GaussianMixture, init_params="random", tied and full covariance) in fp64 on the rounded
//             values.  The row lives in registers, ceil(P/32) values per lane.
//   cross   : fixed-order reduction of the denoising cross-moments over cells: sum z, sum z z^T, sum y_j and
//             sum z y_j, where z = [isotype control columns | bgmean] (q = m+1 columns).
//   apply   : y_ij -= (z_i . w - b) beta_j and/or the quantile clip, one warp per cell.
#include <math.h>

#include <algorithm>

#include "common.cuh"

namespace mub {
namespace dsb {

constexpr int kMomThreads = 256;
constexpr int kMomBlocks = 512;        // fixed: the partial-sum order depends on the input only
constexpr int kMomShared = 32 * 1024;  // row tile of the CSR scatter
constexpr int kFitWarps = 4;
constexpr int kCrossThreads = 256;
constexpr int kCrossRows = 32;         // rows staged per tile
constexpr int kCrossBlocks = 256;
constexpr int kMaxQ = 16;              // isotype controls + 1

constexpr double kReg = 1e-6, kTol = 1e-3;
constexpr int kMaxIter = 100;
constexpr double kEps10 = 10 * 2.220446049250313e-16;
constexpr double kLog2Pi = 1.8378770664093453;  // log(2 pi)
constexpr double kLog2 = 0.6931471805599453;

__device__ __forceinline__ float dlog(float x) { return logf(x); }
__device__ __forceinline__ double dlog(double x) { return log(x); }

// ---- moments ---------------------------------------------------------------------------------------------
template <typename T, bool kCsr>
__global__ void __launch_bounds__(kMomThreads)
moments_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
               const T* __restrict__ data, int64_t n_rows, int P, T pc, int64_t rows_per_block,
               const double* __restrict__ center, double* __restrict__ part) {
    // pass 1 (center == nullptr): sums of d into part[b][0:P]; pass 2: sums of (d - center)^2 into part[b][P:2P]
    extern __shared__ double tile[];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const T l0 = dlog(T(0) + pc);
    const int64_t r0 = (int64_t)blockIdx.x * rows_per_block;
    const int64_t r1 = min(n_rows, r0 + rows_per_block);
    double s1[4] = {0, 0, 0, 0}, s2[4] = {0, 0, 0, 0};
    if (!kCsr) {
        for (int64_t r = r0; r < r1; ++r) {
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const int j = t + c * kMomThreads;
                if (j < P) {
                    const double d = (double)dlog(data[r * P + j] + pc) - (double)l0;
                    if (center) {
                        const double e = d - center[j];
                        s2[c] += e * e;
                    } else {
                        s1[c] += d;
                    }
                }
            }
        }
    } else {
        const int R = max(1, kMomShared / (8 * P));
        for (int j = t; j < R * P; j += kMomThreads) tile[j] = 0.0;
        __syncthreads();
        for (int64_t rb = r0; rb < r1; rb += R) {
            const int nr = (int)min((int64_t)R, r1 - rb);
            for (int rr = warp; rr < nr; rr += kMomThreads / 32) {
                const int64_t s = indptr[rb + rr], e = indptr[rb + rr + 1];
                for (int64_t k = s + lane; k < e; k += 32)
                    tile[rr * P + indices[k]] = (double)dlog(ld_stream(data + k) + pc) - (double)l0;
            }
            __syncthreads();
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const int j = t + c * kMomThreads;
                if (j < P) {
                    const double cj = center ? center[j] : 0.0;
                    for (int rr = 0; rr < nr; ++rr) {
                        const double d = tile[rr * P + j];
                        if (center) {
                            const double e = d - cj;
                            s2[c] += e * e;
                        } else {
                            s1[c] += d;
                        }
                        tile[rr * P + j] = 0.0;
                    }
                }
            }
            __syncthreads();
        }
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const int j = t + c * kMomThreads;
        if (j < P) part[(int64_t)blockIdx.x * 2 * P + (center ? P + j : j)] = center ? s2[c] : s1[c];
    }
}

// block partials added in block order.  After pass 1: mean[j] = log(pc) + mean d and stdev[j] = mean d (the
// centre of pass 2); after pass 2: stdev[j] = sqrt(sum (d - mean d)^2 / (n - 1)) (ddof=1).
template <typename T>
__global__ void moments_finish_kernel(const double* __restrict__ part, int n_blocks, int P, int64_t n_rows, T pc,
                                      bool second, double* __restrict__ mean, double* __restrict__ stdev) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= P) return;
    double s = 0;
    for (int b = 0; b < n_blocks; ++b) s += part[(int64_t)b * 2 * P + (second ? P + j : j)];
    const double n = (double)n_rows;
    if (second) {
        stdev[j] = sqrt(s / (n - 1.0));
    } else {
        mean[j] = (double)dlog(T(0) + pc) + s / n;
        stdev[j] = s / n;
    }
}

// ---- per-cell mixture fits -------------------------------------------------------------------------------
struct Gmm {
    double w0, w1, mu0, mu1, v0, v1;
};

struct FitOut {
    double min_mean, bic;
    int n_iter;
    bool converged;
};

// E-step terms of one value under the current parameters (sklearn _estimate_weighted_log_prob + _logsumexp)
struct EParams {
    double pc0, pc1, mpc0, mpc1, c0, c1;  // precision, mu*precision, log(precision) + log(weight)
};

__device__ __forceinline__ EParams e_params(const Gmm& g) {
    EParams e;
    e.pc0 = 1.0 / sqrt(g.v0);
    e.pc1 = 1.0 / sqrt(g.v1);
    e.mpc0 = g.mu0 * e.pc0;
    e.mpc1 = g.mu1 * e.pc1;
    e.c0 = log(e.pc0);
    e.c1 = log(e.pc1);
    return e;
}

__device__ __forceinline__ double e_value(const EParams& e, double lw0, double lw1, double x, double& r0,
                                          double& r1) {
    const double y0 = x * e.pc0 - e.mpc0, y1 = x * e.pc1 - e.mpc1;
    const double a0 = (-0.5 * (kLog2Pi + y0 * y0) + e.c0) + lw0;
    const double a1 = (-0.5 * (kLog2Pi + y1 * y1) + e.c1) + lw1;
    double lse;
    if (a0 == a1) {
        lse = (0.0 + kLog2) + a0;
    } else {
        const double hi = fmax(a0, a1), lo = fmin(a0, a1);
        lse = (log1p(exp(lo - hi)) + 0.0) + hi;
    }
    r0 = exp(a0 - lse);
    r1 = exp(a1 - lse);
    return lse;
}

template <int V, bool kTied>
__device__ FitOut fit_one(const double (&x)[V], int P, int lane, double xx, const double* __restrict__ u) {
    // initial responsibilities from the uniform draw U (P x 2), then the first M-step (weights nk / P)
    double n0 = 0, n1 = 0, sx0 = 0, sx1 = 0, r0v[V], r1v[V];
#pragma unroll
    for (int v = 0; v < V; ++v) {
        const int j = lane + 32 * v;
        r0v[v] = r1v[v] = 0;
        if (j < P) {
            const double a = u[2 * j], b = u[2 * j + 1], s = a + b;
            r0v[v] = a / s;
            r1v[v] = b / s;
            n0 += r0v[v];
            n1 += r1v[v];
            sx0 += r0v[v] * x[v];
            sx1 += r1v[v] * x[v];
        }
    }
    n0 = warp_sum(n0) + kEps10;
    n1 = warp_sum(n1) + kEps10;
    Gmm g;
    g.mu0 = warp_sum(sx0) / n0;
    g.mu1 = warp_sum(sx1) / n1;
    if (kTied) {
        g.v0 = g.v1 = (xx - (n0 * g.mu0 * g.mu0 + n1 * g.mu1 * g.mu1)) / (n0 + n1) + kReg;
    } else {
        double q0 = 0, q1 = 0;
#pragma unroll
        for (int v = 0; v < V; ++v) {
            const double d0 = x[v] - g.mu0, d1 = x[v] - g.mu1;
            q0 += r0v[v] * d0 * d0;
            q1 += r1v[v] * d1 * d1;
        }
        g.v0 = warp_sum(q0) / n0 + kReg;
        g.v1 = warp_sum(q1) / n1 + kReg;
    }
    g.w0 = n0 / P;
    g.w1 = n1 / P;

    double lower = -INFINITY;
    FitOut out;
    out.converged = false;
    out.n_iter = 0;
    for (int it = 1; it <= kMaxIter; ++it) {
        const EParams e = e_params(g);
        const double lw0 = log(g.w0), lw1 = log(g.w1);
        double sl = 0;
        n0 = n1 = sx0 = sx1 = 0;
#pragma unroll
        for (int v = 0; v < V; ++v) {
            const int j = lane + 32 * v;
            r0v[v] = r1v[v] = 0;
            if (j < P) {
                sl += e_value(e, lw0, lw1, x[v], r0v[v], r1v[v]);
                n0 += r0v[v];
                n1 += r1v[v];
                sx0 += r0v[v] * x[v];
                sx1 += r1v[v] * x[v];
            }
        }
        n0 = warp_sum(n0) + kEps10;
        n1 = warp_sum(n1) + kEps10;
        g.mu0 = warp_sum(sx0) / n0;
        g.mu1 = warp_sum(sx1) / n1;
        if (kTied) {
            g.v0 = g.v1 = (xx - (n0 * g.mu0 * g.mu0 + n1 * g.mu1 * g.mu1)) / (n0 + n1) + kReg;
        } else {
            double q0 = 0, q1 = 0;
#pragma unroll
            for (int v = 0; v < V; ++v) {
                const double d0 = x[v] - g.mu0, d1 = x[v] - g.mu1;
                q0 += r0v[v] * d0 * d0;
                q1 += r1v[v] * d1 * d1;
            }
            g.v0 = warp_sum(q0) / n0 + kReg;
            g.v1 = warp_sum(q1) / n1 + kReg;
        }
        g.w0 = n0 / (n0 + n1);
        g.w1 = n1 / (n0 + n1);
        const double prev = lower;
        lower = warp_sum(sl) / P;
        out.n_iter = it;
        if (fabs(lower - prev) < kTol) {
            out.converged = true;
            break;
        }
    }
    // bic = -2 * score * P + p log P with the final parameters
    const EParams e = e_params(g);
    const double lw0 = log(g.w0), lw1 = log(g.w1);
    double sl = 0, r0, r1;
#pragma unroll
    for (int v = 0; v < V; ++v)
        if (lane + 32 * v < P) sl += e_value(e, lw0, lw1, x[v], r0, r1);
    const double score = warp_sum(sl) / P;
    out.bic = -2 * score * P + (kTied ? 4.0 : 5.0) * log((double)P);
    out.min_mean = fmin(g.mu0, g.mu1);
    return out;
}

template <typename T, int V, bool kCsr>
__global__ void __launch_bounds__(kFitWarps * 32)
fit_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices, const T* __restrict__ data,
           int64_t n_cells, int P, T pc, const double* __restrict__ mean, const double* __restrict__ stdev,
           uint32_t flags, const double* __restrict__ u, int64_t u_cell_stride, int64_t u_model_stride,
           T* __restrict__ out, double* __restrict__ bgmean, int8_t* __restrict__ model,
           int32_t* __restrict__ n_iter, int8_t* __restrict__ converged, int32_t* __restrict__ status) {
    extern __shared__ double rowbuf[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    double* buf = rowbuf + (size_t)wib * P;
    const bool standardize = flags & MUB_DSB_STANDARDIZE, fit = flags & MUB_DSB_FIT;
    for (int64_t cell = (int64_t)blockIdx.x * kFitWarps + wib; cell < n_cells;
         cell += (int64_t)gridDim.x * kFitWarps) {
        T raw[V];
        if (kCsr) {
            for (int j = lane; j < P; j += 32) buf[j] = 0.0;
            __syncwarp();
            const int64_t s = indptr[cell], e = indptr[cell + 1];
            for (int64_t k = s + lane; k < e; k += 32) buf[indices[k]] = (double)ld_stream(data + k);
            __syncwarp();
#pragma unroll
            for (int v = 0; v < V; ++v) {
                const int j = lane + 32 * v;
                raw[v] = j < P ? (T)buf[j] : T(0);
            }
            __syncwarp();
        } else {
#pragma unroll
            for (int v = 0; v < V; ++v) {
                const int j = lane + 32 * v;
                raw[v] = j < P ? ld_stream(data + cell * P + j) : T(0);
            }
        }
        double x[V], xx = 0;
        bool bad = false;
#pragma unroll
        for (int v = 0; v < V; ++v) {
            const int j = lane + 32 * v;
            x[v] = 0;
            if (j < P) {
                double y = (double)dlog(raw[v] + pc) - mean[j];
                if (standardize) y /= stdev[j];
                const T yt = (T)y;
                out[cell * P + j] = yt;
                x[v] = (double)yt;
                bad |= !isfinite(x[v]);
                xx += x[v] * x[v];
            }
        }
        if (!fit) continue;
        if (__any_sync(0xffffffffu, bad)) {
            if (lane == 0) {
                atomicOr(status, 1);
                bgmean[cell] = NAN;
            }
            continue;
        }
        xx = warp_sum(xx);
        const double* uc = u + cell * u_cell_stride;
        const FitOut a = fit_one<V, true>(x, P, lane, xx, uc);
        const FitOut b = fit_one<V, false>(x, P, lane, xx, uc + u_model_stride);
        if (lane == 0) {
            const bool tied = a.bic < b.bic;
            bgmean[cell] = (double)(T)(tied ? a.min_mean : b.min_mean);
            model[cell] = tied ? 0 : 1;
            n_iter[2 * cell] = a.n_iter;
            n_iter[2 * cell + 1] = b.n_iter;
            converged[2 * cell] = a.converged;
            converged[2 * cell + 1] = b.converged;
        }
    }
}

// ---- denoising -------------------------------------------------------------------------------------------
// z_ik: the isotype control columns of the scaled matrix, then bgmean
template <typename T>
__device__ __forceinline__ double z_at(const T* y, int64_t i, int P, const double* bgmean, const int32_t* ctrl,
                                       int k, int q) {
    return k + 1 < q ? (double)y[i * P + ctrl[k]] : bgmean[i];
}

// partial sums per block: [sum z (q) | sum z z^T (q*q) | sum y (P) | sum z y^T (q*P)]
template <typename T, int Q>
__global__ void __launch_bounds__(kCrossThreads)
cross_kernel(const T* __restrict__ y, int64_t n, int P, const double* __restrict__ bgmean,
             const int32_t* __restrict__ ctrl, int q, int64_t rows_per_block, double* __restrict__ part) {
    __shared__ double zt[kCrossRows][kMaxQ];
    const int t = threadIdx.x;
    const int j = blockIdx.y * kCrossThreads + t;
    const int64_t r0 = (int64_t)blockIdx.x * rows_per_block, r1 = min(n, r0 + rows_per_block);
    const int64_t S = q + q * q + P + (int64_t)q * P;
    double sy = 0, szy[Q], sm = 0;  // sm: this thread's entry of sum z / sum z z^T (block column 0 only)
#pragma unroll
    for (int k = 0; k < Q; ++k) szy[k] = 0;
    const bool mom = blockIdx.y == 0 && t < q + q * q;
    const int mk = t < q ? t : (t - q) / q, ml = t < q ? -1 : (t - q) % q;
    for (int64_t rb = r0; rb < r1; rb += kCrossRows) {
        const int nr = (int)min((int64_t)kCrossRows, r1 - rb);
        __syncthreads();
        for (int e = t; e < nr * q; e += kCrossThreads)
            zt[e / q][e % q] = z_at(y, rb + e / q, P, bgmean, ctrl, e % q, q);
        __syncthreads();
        if (j < P) {
            for (int rr = 0; rr < nr; ++rr) {
                const double v = (double)y[(rb + rr) * P + j];
                sy += v;
#pragma unroll
                for (int k = 0; k < Q; ++k)
                    if (k < q) szy[k] += zt[rr][k] * v;
            }
        }
        if (mom)
            for (int rr = 0; rr < nr; ++rr) sm += ml < 0 ? zt[rr][mk] : zt[rr][mk] * zt[rr][ml];
    }
    double* p = part + (int64_t)blockIdx.x * S;
    if (mom) p[t] = sm;
    if (j < P) {
        p[q + q * q + j] = sy;
#pragma unroll
        for (int k = 0; k < Q; ++k)
            if (k < q) p[q + q * q + P + (int64_t)k * P + j] = szy[k];
    }
}

__global__ void sum_partials_kernel(const double* __restrict__ part, int n_blocks, int64_t S,
                                    double* __restrict__ out) {
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    double acc = 0;
    for (int b = 0; b < n_blocks; ++b) acc += part[(int64_t)b * S + s];
    out[s] = acc;
}

template <typename T>
__global__ void __launch_bounds__(256)
apply_kernel(T* __restrict__ y, int64_t n, int P, const double* __restrict__ bgmean,
             const int32_t* __restrict__ ctrl, int q, const double* __restrict__ w, double b,
             const double* __restrict__ beta, double lo, double hi, uint32_t flags) {
    const int lane = threadIdx.x & 31;
    const bool clip = flags & MUB_DSB_CLIP;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n;
         i += ((int64_t)gridDim.x * blockDim.x) >> 5) {
        double c = 0;
        if (beta) {
            double zc = lane < q ? z_at(y, i, P, bgmean, ctrl, lane, q) * w[lane] : 0.0;
            c = warp_sum(zc) - b;
        }
        __syncwarp();  // every lane has read its control value before any lane writes the row
        for (int j = lane; j < P; j += 32) {
            double v = (double)y[i * P + j];
            if (beta) v -= c * beta[j];
            if (clip) v = fmin(fmax(v, lo), hi);
            y[i * P + j] = (T)v;
        }
    }
}

// ---- host wrappers ---------------------------------------------------------------------------------------
inline int mom_blocks(int64_t n_rows) { return (int)std::min<int64_t>(kMomBlocks, std::max<int64_t>(1, n_rows)); }

template <typename T>
int moments(const int64_t* indptr, const int32_t* indices, const T* data, int64_t n_rows, int32_t P, T pc,
            void* workspace, double* mean, double* stdev, mub_stream_t stream) {
    MUB_REQUIRE(P >= 1 && P <= MUB_DSB_MAX_PROTEINS, "dsb: %d proteins (1..%d supported)", P,
                MUB_DSB_MAX_PROTEINS);
    MUB_REQUIRE(n_rows >= 0 && data && workspace && mean && stdev, "dsb moments: bad arguments");
    cudaStream_t s = (cudaStream_t)stream;
    const int G = mom_blocks(n_rows);
    const int64_t rpb = (n_rows + G - 1) / G;
    double* part = (double*)workspace;
    MUB_REQUIRE(!indptr || indices, "dsb moments: CSR without indices");
    for (int pass = 0; pass < 2; ++pass) {
        const double* center = pass ? stdev : nullptr;
        if (indptr)
            moments_kernel<T, true><<<G, kMomThreads, kMomShared, s>>>(indptr, indices, data, n_rows, P, pc, rpb,
                                                                       center, part);
        else
            moments_kernel<T, false><<<G, kMomThreads, 0, s>>>(indptr, indices, data, n_rows, P, pc, rpb, center,
                                                               part);
        if (int rc = check_launch("dsb_moments_kernel")) return rc;
        moments_finish_kernel<T><<<(P + 127) / 128, 128, 0, s>>>(part, G, P, n_rows, pc, pass == 1, mean, stdev);
        if (int rc = check_launch("dsb_moments_finish_kernel")) return rc;
    }
    return 0;
}

template <typename T, int V>
int fit_v(const int64_t* indptr, const int32_t* indices, const T* data, int64_t n, int P, T pc,
          const double* mean, const double* stdev, uint32_t flags, const double* u, int64_t ucs, int64_t ums,
          T* out, double* bg, int8_t* model, int32_t* n_iter, int8_t* conv, int32_t* status, cudaStream_t s) {
    const int64_t want = (n + kFitWarps - 1) / kFitWarps;
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(want, (int64_t)sm_count() * 64));
    if (indptr) {
        const size_t smem = (size_t)kFitWarps * P * sizeof(double);
        fit_kernel<T, V, true><<<grid, kFitWarps * 32, smem, s>>>(indptr, indices, data, n, P, pc, mean, stdev,
                                                                 flags, u, ucs, ums, out, bg, model, n_iter,
                                                                 conv, status);
    } else {
        fit_kernel<T, V, false><<<grid, kFitWarps * 32, 0, s>>>(indptr, indices, data, n, P, pc, mean, stdev,
                                                               flags, u, ucs, ums, out, bg, model, n_iter,
                                                               conv, status);
    }
    return check_launch("dsb_fit_kernel");
}

template <typename T>
int fit(const int64_t* indptr, const int32_t* indices, const T* data, int64_t n, int32_t P, T pc,
        const double* mean, const double* stdev, uint32_t flags, const double* u, int64_t ucs, int64_t ums,
        T* out, double* bg, int8_t* model, int32_t* n_iter, int8_t* conv, int32_t* status,
        mub_stream_t stream) {
    MUB_REQUIRE(P >= 1 && P <= MUB_DSB_MAX_PROTEINS, "dsb: %d proteins (1..%d supported)", P,
                MUB_DSB_MAX_PROTEINS);
    MUB_REQUIRE(n >= 0 && data && mean && stdev && out, "dsb fit: bad arguments");
    MUB_REQUIRE(!(flags & MUB_DSB_FIT) || (P >= 2 && u && bg && model && n_iter && conv && status),
                "dsb fit: the mixture fits need P >= 2, the draws and every per-cell output");
    if (n == 0) return 0;
    cudaStream_t s = (cudaStream_t)stream;
#define MUB_DSB_FIT_V(V) \
    return fit_v<T, V>(indptr, indices, data, n, P, pc, mean, stdev, flags, u, ucs, ums, out, bg, model, n_iter, \
                       conv, status, s)
    if (P <= 32) MUB_DSB_FIT_V(1);
    if (P <= 64) MUB_DSB_FIT_V(2);
    if (P <= 128) MUB_DSB_FIT_V(4);
    if (P <= 256) MUB_DSB_FIT_V(8);
    if (P <= 512) MUB_DSB_FIT_V(16);
    MUB_DSB_FIT_V(32);
#undef MUB_DSB_FIT_V
}

inline int cross_blocks(int64_t n) { return (int)std::min<int64_t>(kCrossBlocks, std::max<int64_t>(1, (n + 255) / 256)); }

template <typename T>
int cross(const T* y, int64_t n, int32_t P, const double* bgmean, const int32_t* ctrl, int32_t m,
          void* workspace, double* sums, mub_stream_t stream) {
    const int q = m + 1;
    MUB_REQUIRE(P >= 1 && P <= MUB_DSB_MAX_PROTEINS && m >= 0 && q <= MUB_DSB_MAX_CONTROLS + 1,
                "dsb cross: P=%d, %d controls (at most %d)", P, m, MUB_DSB_MAX_CONTROLS);
    MUB_REQUIRE(y && bgmean && workspace && sums && (m == 0 || ctrl), "dsb cross: bad arguments");
    cudaStream_t s = (cudaStream_t)stream;
    const int G = cross_blocks(n);
    const int64_t rpb = (n + G - 1) / G;
    const int64_t S = q + q * q + P + (int64_t)q * P;
    double* part = (double*)workspace;
    const dim3 grid(G, (P + kCrossThreads - 1) / kCrossThreads);
    if (q <= 1)
        cross_kernel<T, 1><<<grid, kCrossThreads, 0, s>>>(y, n, P, bgmean, ctrl, q, rpb, part);
    else if (q <= 4)
        cross_kernel<T, 4><<<grid, kCrossThreads, 0, s>>>(y, n, P, bgmean, ctrl, q, rpb, part);
    else
        cross_kernel<T, kMaxQ><<<grid, kCrossThreads, 0, s>>>(y, n, P, bgmean, ctrl, q, rpb, part);
    if (int rc = check_launch("dsb_cross_kernel")) return rc;
    sum_partials_kernel<<<(unsigned)((S + 255) / 256), 256, 0, s>>>(part, G, S, sums);
    return check_launch("dsb_sum_partials_kernel");
}

template <typename T>
int apply(T* y, int64_t n, int32_t P, const double* bgmean, const int32_t* ctrl, int32_t m, const double* w,
          double b, const double* beta, double lo, double hi, uint32_t flags, mub_stream_t stream) {
    MUB_REQUIRE(P >= 1 && m >= 0 && m + 1 <= 32 && y, "dsb apply: bad arguments");
    MUB_REQUIRE(!beta || (bgmean && w && (m == 0 || ctrl)), "dsb apply: the denoising term needs bgmean and w");
    if (n == 0) return 0;
    const int64_t want = (n * 32 + 255) / 256;
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(want, (int64_t)sm_count() * 16));
    apply_kernel<T><<<grid, 256, 0, (cudaStream_t)stream>>>(y, n, P, bgmean, ctrl, m + 1, w, b, beta, lo, hi,
                                                            flags);
    return check_launch("dsb_apply_kernel");
}

}  // namespace dsb
}  // namespace mub

extern "C" {

size_t mub_dsb_moments_workspace_bytes(int64_t n_rows, int32_t n_prot) {
    return (size_t)mub::dsb::mom_blocks(n_rows) * 2 * (size_t)n_prot * sizeof(double);
}

int mub_dsb_moments_f32(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_rows,
                        int32_t n_prot, float pseudocount, void* workspace, double* mean, double* stdev,
                        mub_stream_t stream) {
    return mub::dsb::moments<float>(indptr, indices, data, n_rows, n_prot, pseudocount, workspace, mean, stdev,
                                    stream);
}
int mub_dsb_moments_f64(const int64_t* indptr, const int32_t* indices, const double* data, int64_t n_rows,
                        int32_t n_prot, double pseudocount, void* workspace, double* mean, double* stdev,
                        mub_stream_t stream) {
    return mub::dsb::moments<double>(indptr, indices, data, n_rows, n_prot, pseudocount, workspace, mean, stdev,
                                     stream);
}

int mub_dsb_fit_f32(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_cells,
                    int32_t n_prot, float pseudocount, const double* mean, const double* stdev, uint32_t flags,
                    const double* draws, int64_t draw_cell_stride, int64_t draw_model_stride, float* out,
                    double* bgmean, int8_t* model, int32_t* n_iter, int8_t* converged, int32_t* status,
                    mub_stream_t stream) {
    return mub::dsb::fit<float>(indptr, indices, data, n_cells, n_prot, pseudocount, mean, stdev, flags, draws,
                                draw_cell_stride, draw_model_stride, out, bgmean, model, n_iter, converged,
                                status, stream);
}
int mub_dsb_fit_f64(const int64_t* indptr, const int32_t* indices, const double* data, int64_t n_cells,
                    int32_t n_prot, double pseudocount, const double* mean, const double* stdev, uint32_t flags,
                    const double* draws, int64_t draw_cell_stride, int64_t draw_model_stride, double* out,
                    double* bgmean, int8_t* model, int32_t* n_iter, int8_t* converged, int32_t* status,
                    mub_stream_t stream) {
    return mub::dsb::fit<double>(indptr, indices, data, n_cells, n_prot, pseudocount, mean, stdev, flags, draws,
                                 draw_cell_stride, draw_model_stride, out, bgmean, model, n_iter, converged,
                                 status, stream);
}

size_t mub_dsb_cross_workspace_bytes(int64_t n_cells, int32_t n_prot, int32_t n_controls) {
    const int64_t q = n_controls + 1;
    return (size_t)mub::dsb::cross_blocks(n_cells) * (size_t)(q + q * q + n_prot + q * n_prot) * sizeof(double);
}

int mub_dsb_cross_f32(const float* y, int64_t n_cells, int32_t n_prot, const double* bgmean,
                      const int32_t* controls, int32_t n_controls, void* workspace, double* sums,
                      mub_stream_t stream) {
    return mub::dsb::cross<float>(y, n_cells, n_prot, bgmean, controls, n_controls, workspace, sums, stream);
}
int mub_dsb_cross_f64(const double* y, int64_t n_cells, int32_t n_prot, const double* bgmean,
                      const int32_t* controls, int32_t n_controls, void* workspace, double* sums,
                      mub_stream_t stream) {
    return mub::dsb::cross<double>(y, n_cells, n_prot, bgmean, controls, n_controls, workspace, sums, stream);
}

int mub_dsb_apply_f32(float* y, int64_t n_cells, int32_t n_prot, const double* bgmean, const int32_t* controls,
                      int32_t n_controls, const double* w, double b, const double* beta, double lo, double hi,
                      uint32_t flags, mub_stream_t stream) {
    return mub::dsb::apply<float>(y, n_cells, n_prot, bgmean, controls, n_controls, w, b, beta, lo, hi, flags,
                                  stream);
}
int mub_dsb_apply_f64(double* y, int64_t n_cells, int32_t n_prot, const double* bgmean, const int32_t* controls,
                      int32_t n_controls, const double* w, double b, const double* beta, double lo, double hi,
                      uint32_t flags, mub_stream_t stream) {
    return mub::dsb::apply<double>(y, n_cells, n_prot, bgmean, controls, n_controls, w, b, beta, lo, hi, flags,
                                   stream);
}

}  // extern "C"
