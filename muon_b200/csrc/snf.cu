// K13 -- similarity network fusion (Wang et al. 2014) as muon.tl.snf computes it, float64 throughout.
//
//   The fused state of each modality is kept as a raw bit-symmetric N x N matrix X plus its row sums minus the
//   diagonal r (0 replaced by 1).  The normalised matrix of the reference's _normalize is never stored: every reader
//   applies
//       nv(X)[i, j] = 0.5                                        if i == j
//                   = (X[i,j] / (2 r[i]) + X[i,j] / (2 r[j])) / 2  otherwise,
//   which is the reference's (x / (2 r) with diagonal 0.5, then (x + x^T) / 2) for a bit-symmetric x, and is itself
//   bit-symmetric because the sum of the two halves commutes.
//
//   Kernels:
//     symmetrise_kernel   (D + D^T) / 2 with a zero diagonal, in place, one 32 x 32 tile pair per block;
//     densify_kernel      a canonical CSR of distances as a dense matrix: unstored = +inf, diagonal 0;
//     select_kernel       per-row k smallest / largest with ties broken by ascending column: an 8 x 8-bit radix
//                         select of the order-preserving key, one index-order collection pass, a bitonic sort of
//                         the k survivors; one block per row;
//     means_kernel, affinity_kernel   finite mean of sorted positions 1..k, then the scaled normal pdf;
//     rowsum_kernel       r[i] = sum_j X[i,j] - X[i,i] (0 -> 1), fixed reduction tree;
//     average_kernel      (nv(X_0) + nv(X_1) + ...) / div, summed in the order given;
//     colsum/scale kernels  the dominate set's column sums over the transposed top-k structure, and S = T^T / cs;
//     diffuse_kernel      one 64 x 64 output tile of S . B, B read with nv on the fly; written transposed
//                         (R^T = (S P)^T), or as the upper triangle of S . R^T mirrored into the lower one so that
//                         nextW = S P S^T comes out bit-symmetric.  Every sum runs in a fixed order: no atomics
//                         touch a float, so each call returns the same bits.
#include <math.h>

#include "common.cuh"

namespace mub {
namespace snf {

constexpr int kThreads = 256;
constexpr int kTile = 64;                              // diffusion tile edge
constexpr int kSymTile = 32;                           // symmetrise tile edge
constexpr int kSelCap = MUB_SNF_MAX_NEIGHBORS + 1;     // the means selection takes k + 1 entries
static_assert(kSelCap <= kThreads, "one bitonic slot per thread");

struct Mods {
    const double* x[MUB_SNF_MAX_MODALITIES];
    const double* r[MUB_SNF_MAX_MODALITIES];
};

__device__ __forceinline__ double nv(double x, int64_t i, int64_t j, const double* __restrict__ r) {
    if (r == nullptr) return x;
    if (i == j) return 0.5;
    const double a = x / (2.0 * r[i]);
    const double b = x / (2.0 * r[j]);
    return (a + b) / 2.0;
}

// ---- (D + D^T) / 2, zero diagonal ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(kSymTile * 8) symmetrise_kernel(double* D, int64_t n) {
    const int ti = blockIdx.y, tj = blockIdx.x;
    if (ti > tj) return;
    __shared__ double A[kSymTile][kSymTile + 1], B[kSymTile][kSymTile + 1];
    const int tx = threadIdx.x % kSymTile, ty = threadIdx.x / kSymTile;
    const int64_t i0 = (int64_t)ti * kSymTile, j0 = (int64_t)tj * kSymTile;
    for (int y = ty; y < kSymTile; y += 8) {
        const int64_t ia = i0 + y, ja = j0 + tx, ib = j0 + y, jb = i0 + tx;
        A[y][tx] = ia < n && ja < n ? D[ia * n + ja] : 0.0;
        B[y][tx] = ib < n && jb < n ? D[ib * n + jb] : 0.0;
    }
    __syncthreads();
    for (int y = ty; y < kSymTile; y += 8) {
        const int64_t ia = i0 + y, ja = j0 + tx, ib = j0 + y, jb = i0 + tx;
        if (ia < n && ja < n) D[ia * n + ja] = ia == ja ? 0.0 : (A[y][tx] + B[tx][y]) / 2.0;
        if (ib < n && jb < n) D[ib * n + jb] = ib == jb ? 0.0 : (B[y][tx] + A[tx][y]) / 2.0;
    }
}

// ---- canonical CSR -> dense, unstored = +inf ----------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) densify_kernel(const int64_t* __restrict__ indptr,
                                                           const int32_t* __restrict__ indices,
                                                           const double* __restrict__ data, int64_t n, double* out) {
    const int64_t i = blockIdx.x;
    double* row = out + i * n;
    for (int64_t j = threadIdx.x; j < n; j += kThreads) row[j] = j == i ? 0.0 : (double)INFINITY;
    __syncthreads();
    for (int64_t e = indptr[i] + threadIdx.x; e < indptr[i + 1]; e += kThreads) {
        const int64_t j = indices[e];
        if (j != i) row[j] = data[e];
    }
}

// ---- row selection ------------------------------------------------------------------------------------------------
__device__ __forceinline__ double select_value(const double* __restrict__ row, int64_t i, int64_t j,
                                               const double* __restrict__ r, int mode) {
    const double x = nv(row[j], i, j, r);
    return mode == MUB_SNF_SELECT_DIST ? 0.5 - x : x;
}

__device__ __forceinline__ bool select_valid(double v, int mode) {
    return !(mode == MUB_SNF_SELECT_DIST || mode == MUB_SNF_SELECT_CONN) || v != 0.0;
}

// order-preserving key: ascending for the smallest modes, descending for the largest; -0 is folded into +0
__device__ __forceinline__ uint64_t select_key(double v, int mode) {
    uint64_t b = (uint64_t)__double_as_longlong(v + 0.0);
    b = (b >> 63) ? ~b : (b | 0x8000000000000000ull);
    return mode == MUB_SNF_SELECT_LARGEST ? ~b : b;
}

__global__ void __launch_bounds__(kThreads) select_kernel(const double* __restrict__ X, const double* __restrict__ r,
                                                          int64_t n, int k, int mode, int32_t* __restrict__ out_idx,
                                                          double* __restrict__ out_val, int32_t* __restrict__ out_cnt) {
    const int64_t i = blockIdx.x;
    const double* row = X + i * n;
    const int lane = threadIdx.x % kWarp, warp = threadIdx.x / kWarp;
    constexpr int kWarps = kThreads / kWarp;
    __shared__ int hist[256];
    __shared__ int s_remaining, s_total, s_digit;
    __shared__ int s_wl[kWarps], s_wt[kWarps];
    __shared__ uint64_t s_key[kSelCap <= 128 ? 128 : 256];
    __shared__ int32_t s_idx[kSelCap <= 128 ? 128 : 256];
    constexpr int kSort = kSelCap <= 128 ? 128 : 256;

    uint64_t prefix = 0, mask = 0;
    int remaining = 0;
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (int q = threadIdx.x; q < 256; q += kThreads) hist[q] = 0;
        __syncthreads();
        for (int64_t j = threadIdx.x; j < n; j += kThreads) {
            const double v = select_value(row, i, j, r, mode);
            if (!select_valid(v, mode)) continue;
            const uint64_t key = select_key(v, mode);
            if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255], 1);
        }
        __syncthreads();
        if (warp == 0) {
            const int prev = s_remaining;
            int c[8], s = 0;
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                c[q] = hist[lane * 8 + q];
                s += c[q];
            }
            int incl = s;
#pragma unroll
            for (int o = 1; o < kWarp; o <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += t;
            }
            const int total = __shfl_sync(0xffffffffu, incl, kWarp - 1);
            int want;
            if (shift == 56) {
                want = min(k, total);
                if (lane == 0) s_total = want;
            } else {
                want = prev;
            }
            __syncwarp();
            const int excl = incl - s;
            if (want > 0 && excl < want && want <= incl) {
                int acc = excl;
                for (int q = 0; q < 8; ++q) {
                    if (acc + c[q] >= want) {
                        s_digit = lane * 8 + q;
                        s_remaining = want - acc;
                        break;
                    }
                    acc += c[q];
                }
            }
            if (want == 0 && lane == 0) {
                s_digit = 0;
                s_remaining = 0;
            }
        }
        __syncthreads();
        prefix |= (uint64_t)s_digit << shift;
        mask |= (uint64_t)255 << shift;
        remaining = s_remaining;
        __syncthreads();
    }
    const int kk = s_total;
    const int need_ties = remaining;             // entries equal to the threshold key that are kept
    const int n_less = kk - need_ties;           // entries strictly below it
    // collection in ascending column order: every smaller key, then the first need_ties equal keys
    int base_less = 0, base_tie = 0;
    for (int64_t c0 = 0; c0 < n && kk > 0; c0 += kThreads) {
        const int64_t j = c0 + threadIdx.x;
        bool less = false, tie = false;
        if (j < n) {
            const double v = select_value(row, i, j, r, mode);
            if (select_valid(v, mode)) {
                const uint64_t key = select_key(v, mode);
                less = key < prefix;
                tie = key == prefix;
            }
        }
        const unsigned bl = __ballot_sync(0xffffffffu, less), bt = __ballot_sync(0xffffffffu, tie);
        const unsigned lt = (1u << lane) - 1u;
        if (lane == 0) {
            s_wl[warp] = __popc(bl);
            s_wt[warp] = __popc(bt);
        }
        __syncthreads();
        int off_l = base_less, off_t = base_tie, tot_l = base_less, tot_t = base_tie;
        for (int w = 0; w < kWarps; ++w) {
            if (w < warp) {
                off_l += s_wl[w];
                off_t += s_wt[w];
            }
            tot_l += s_wl[w];
            tot_t += s_wt[w];
        }
        if (less) {
            const int p = off_l + __popc(bl & lt);
            s_key[p] = select_key(select_value(row, i, j, r, mode), mode);
            s_idx[p] = (int32_t)j;
        }
        if (tie) {
            const int t = off_t + __popc(bt & lt);
            if (t < need_ties) {
                s_key[n_less + t] = prefix;
                s_idx[n_less + t] = (int32_t)j;
            }
        }
        base_less = tot_l;
        base_tie = tot_t;
        __syncthreads();
        if (base_less >= n_less && base_tie >= need_ties) break;
    }
    for (int p = kk + threadIdx.x; p < kSort; p += kThreads) {
        s_key[p] = ~0ull;
        s_idx[p] = 0x7fffffff;
    }
    __syncthreads();
    // bitonic sort of (key, column)
    for (int size = 2; size <= kSort; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            const int p = threadIdx.x;
            if (p < kSort) {
                const int q = p ^ stride;
                if (q > p) {
                    const bool up = (p & size) == 0;
                    const uint64_t kp = s_key[p], kq = s_key[q];
                    const int32_t ip = s_idx[p], iq = s_idx[q];
                    const bool gt = kp > kq || (kp == kq && ip > iq);
                    if (gt == up) {
                        s_key[p] = kq;
                        s_key[q] = kp;
                        s_idx[p] = iq;
                        s_idx[q] = ip;
                    }
                }
            }
            __syncthreads();
        }
    }
    for (int p = threadIdx.x; p < k; p += kThreads) {
        if (p < kk) {
            const int32_t j = s_idx[p];
            out_idx[i * k + p] = j;
            out_val[i * k + p] = select_value(row, i, j, r, mode);
        } else {
            out_idx[i * k + p] = -1;
            out_val[i * k + p] = 0.0;
        }
    }
    if (threadIdx.x == 0 && out_cnt != nullptr) out_cnt[i] = kk;
}

// ---- affinity -----------------------------------------------------------------------------------------------------
__global__ void means_kernel(const double* __restrict__ sel, int64_t n, int k, double eps, double* __restrict__ means) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double s = 0.0;
    int c = 0;
    for (int p = 1; p <= k; ++p) {
        const double v = sel[i * (k + 1) + p];
        if (!isinf(v)) {
            s += v;
            ++c;
        }
    }
    means[i] = s / (double)c + eps;
}

__global__ void __launch_bounds__(kThreads) affinity_kernel(double* D, int64_t n, const double* __restrict__ means,
                                                            double sigma, double eps) {
    const int64_t i = blockIdx.x;
    const double mi = means[i];
    const double kRootTwoPi = 2.5066282746310002;   // sqrt(2 pi) as numpy rounds it
    double* row = D + i * n;
    for (int64_t j = threadIdx.x; j < n; j += kThreads) {
        const double d = row[j];
        double w = 0.0;
        if (!isinf(d)) {
            const double sig = (mi + means[j]) / 3.0 + d / 3.0 + eps;
            const double scale = sigma * sig;
            const double y = d / scale;
            w = exp(-(y * y) / 2.0) / kRootTwoPi / scale;
        }
        row[j] = w;
    }
}

// ---- row sums, averages -------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) rowsum_kernel(const double* __restrict__ X, int64_t n, double* r) {
    const int64_t i = blockIdx.x;
    const double* row = X + i * n;
    double s = 0.0;
    for (int64_t j = threadIdx.x; j < n; j += kThreads) s += row[j];
    s = warp_sum(s);
    __shared__ double ws[kThreads / kWarp];
    if (threadIdx.x % kWarp == 0) ws[threadIdx.x / kWarp] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < kThreads / kWarp; ++w) t += ws[w];
        t -= row[i];
        r[i] = t == 0.0 ? 1.0 : t;
    }
}

__global__ void __launch_bounds__(kThreads) average_kernel(Mods m, int count, double div, int64_t n, double* out) {
    const int64_t i = blockIdx.x;
    for (int64_t j = threadIdx.x; j < n; j += kThreads) {
        double s = 0.0;
        for (int q = 0; q < count; ++q) s += nv(m.x[q][i * n + j], i, j, m.r[q]);
        out[i * n + j] = s / div;
    }
}

// ---- dominate set -------------------------------------------------------------------------------------------------
__global__ void colsum_kernel(const int64_t* __restrict__ ptr, const double* __restrict__ val, int64_t n,
                              double* __restrict__ cs) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double s = 0.0;
    for (int64_t e = ptr[i]; e < ptr[i + 1]; ++e) s += val[e];
    cs[i] = s;
}

__global__ void scale_kernel(const int64_t* __restrict__ ptr, const int32_t* __restrict__ col,
                             const double* __restrict__ val, int64_t n, const double* __restrict__ cs,
                             double* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    for (int64_t e = ptr[i]; e < ptr[i + 1]; ++e) out[e] = val[e] / cs[col[e]];
}

// ---- diffusion: one 64 x 64 tile of S . B ------------------------------------------------------------------------
template <bool kSym>
__global__ void __launch_bounds__(kThreads, 3) diffuse_kernel(const int64_t* __restrict__ sp,
                                                           const int32_t* __restrict__ sc,
                                                           const double* __restrict__ sv, int64_t n,
                                                           const double* __restrict__ B,
                                                           const double* __restrict__ rB, double* __restrict__ out) {
    const int ti = blockIdx.y, tj = blockIdx.x;
    if (kSym && ti > tj) return;
    __shared__ double t[kTile][kTile + 1];
    const int lane = threadIdx.x % kWarp, warp = threadIdx.x / kWarp;
    const int64_t i0 = (int64_t)ti * kTile, c0 = (int64_t)tj * kTile;
    const int64_t ca = c0 + lane, cb = c0 + lane + kWarp;
    const bool va = ca < n, vb = cb < n;
    const double ra = rB != nullptr && va ? rB[ca] : 1.0, rb = rB != nullptr && vb ? rB[cb] : 1.0;
    constexpr int kRows = kTile / (kThreads / kWarp);
    for (int q = 0; q < kRows; ++q) {
        const int y = warp * kRows + q;
        const int64_t i = i0 + y;
        double acc0 = 0.0, acc1 = 0.0;
        if (i < n) {
            const int64_t e0 = sp[i], e1 = sp[i + 1];
            int64_t e = e0;
            for (; e + 4 <= e1; e += 4) {
                int64_t a[4];
                double s[4], b0[4], b1[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    a[u] = __ldg(sc + e + u);
                    s[u] = __ldg(sv + e + u);
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    b0[u] = va ? __ldg(B + a[u] * n + ca) : 0.0;
                    b1[u] = vb ? __ldg(B + a[u] * n + cb) : 0.0;
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    if (rB != nullptr) {
                        const double rr = __ldg(rB + a[u]);
                        b0[u] = a[u] == ca ? 0.5 : (b0[u] / (2.0 * rr) + b0[u] / (2.0 * ra)) / 2.0;
                        b1[u] = a[u] == cb ? 0.5 : (b1[u] / (2.0 * rr) + b1[u] / (2.0 * rb)) / 2.0;
                    }
                    acc0 = fma(s[u], b0[u], acc0);
                    acc1 = fma(s[u], b1[u], acc1);
                }
            }
            for (; e < e1; ++e) {
                const int64_t a = __ldg(sc + e);
                const double s = __ldg(sv + e);
                double b0 = va ? __ldg(B + a * n + ca) : 0.0, b1 = vb ? __ldg(B + a * n + cb) : 0.0;
                if (rB != nullptr) {
                    const double rr = __ldg(rB + a);
                    b0 = a == ca ? 0.5 : (b0 / (2.0 * rr) + b0 / (2.0 * ra)) / 2.0;
                    b1 = a == cb ? 0.5 : (b1 / (2.0 * rr) + b1 / (2.0 * rb)) / 2.0;
                }
                acc0 = fma(s, b0, acc0);
                acc1 = fma(s, b1, acc1);
            }
        }
        t[y][lane] = acc0;
        t[y][lane + kWarp] = acc1;
    }
    __syncthreads();
    if (kSym) {
        // out[I, J] row-major; the diagonal tile takes its lower half from the upper one
        for (int q = 0; q < kRows; ++q) {
            const int y = warp * kRows + q;
            const int64_t i = i0 + y;
            if (i >= n) continue;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int x = lane + h * kWarp;
                const int64_t c = c0 + x;
                if (c >= n) continue;
                out[i * n + c] = (ti == tj && x < y) ? t[x][y] : t[y][x];
            }
        }
        if (ti == tj) return;
    }
    // out[J, I] = tile^T
    for (int q = 0; q < kRows; ++q) {
        const int x = warp * kRows + q;   // column of the tile = row of the output
        const int64_t c = c0 + x;
        if (c >= n) continue;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int y = lane + h * kWarp;
            const int64_t i = i0 + y;
            if (i < n) out[c * n + i] = t[y][x];
        }
    }
}

inline unsigned row_blocks(int64_t n) { return (unsigned)n; }

}  // namespace snf
}  // namespace mub

using namespace mub::snf;

extern "C" int mub_snf_symmetrise_f64(double* D, int64_t n, mub_stream_t stream) {
    MUB_REQUIRE(n >= 1 && n <= MUB_SNF_MAX_CELLS, "snf: %lld cells", (long long)n);
    const unsigned t = (unsigned)((n + kSymTile - 1) / kSymTile);
    symmetrise_kernel<<<dim3(t, t), kSymTile * 8, 0, (cudaStream_t)stream>>>(D, n);
    return mub::check_launch("snf_symmetrise");
}

extern "C" int mub_snf_densify_f64(const int64_t* indptr, const int32_t* indices, const double* data, int64_t n,
                                   double* out, mub_stream_t stream) {
    MUB_REQUIRE(n >= 1 && n <= MUB_SNF_MAX_CELLS, "snf: %lld cells", (long long)n);
    densify_kernel<<<row_blocks(n), kThreads, 0, (cudaStream_t)stream>>>(indptr, indices, data, n, out);
    return mub::check_launch("snf_densify");
}

extern "C" int mub_snf_select_f64(const double* X, const double* r, int64_t n, int32_t k, int32_t mode,
                                  int32_t* out_idx, double* out_val, int32_t* out_count, mub_stream_t stream) {
    MUB_REQUIRE(n >= 1 && n <= MUB_SNF_MAX_CELLS, "snf: %lld cells", (long long)n);
    MUB_REQUIRE(k >= 1 && k <= kSelCap, "snf: selection of %d entries outside [1, %d]", k, kSelCap);
    MUB_REQUIRE(mode >= MUB_SNF_SELECT_SMALLEST && mode <= MUB_SNF_SELECT_CONN, "snf: selection mode %d", mode);
    MUB_REQUIRE(mode == MUB_SNF_SELECT_SMALLEST || r != nullptr, "snf: selection mode %d needs row sums", mode);
    select_kernel<<<row_blocks(n), kThreads, 0, (cudaStream_t)stream>>>(
        X, mode == MUB_SNF_SELECT_SMALLEST ? nullptr : r, n, k, mode, out_idx, out_val, out_count);
    return mub::check_launch("snf_select");
}

extern "C" int mub_snf_affinity_f64(double* D, int64_t n, const double* sel, int32_t k, double sigma, double eps,
                                    double* means, mub_stream_t stream) {
    MUB_REQUIRE(n >= 1 && n <= MUB_SNF_MAX_CELLS, "snf: %lld cells", (long long)n);
    MUB_REQUIRE(k >= 1 && k < kSelCap, "snf: k = %d", k);
    cudaStream_t st = (cudaStream_t)stream;
    means_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(sel, n, k, eps, means);
    affinity_kernel<<<row_blocks(n), kThreads, 0, st>>>(D, n, means, sigma, eps);
    return mub::check_launch("snf_affinity");
}

extern "C" int mub_snf_rowsum_f64(const double* X, int64_t n, double* r, mub_stream_t stream) {
    MUB_REQUIRE(n >= 1 && n <= MUB_SNF_MAX_CELLS, "snf: %lld cells", (long long)n);
    rowsum_kernel<<<row_blocks(n), kThreads, 0, (cudaStream_t)stream>>>(X, n, r);
    return mub::check_launch("snf_rowsum");
}

extern "C" int mub_snf_average_f64(const double* const* xs, const double* const* rs, int32_t count, double div,
                                   int64_t n, double* out, mub_stream_t stream) {
    MUB_REQUIRE(n >= 1 && n <= MUB_SNF_MAX_CELLS, "snf: %lld cells", (long long)n);
    MUB_REQUIRE(count >= 1 && count <= MUB_SNF_MAX_MODALITIES, "snf: %d matrices to average", count);
    Mods m{};
    for (int q = 0; q < count; ++q) {
        m.x[q] = xs[q];
        m.r[q] = rs[q];
        MUB_REQUIRE(xs[q] != out || count == 1, "snf: an average of several matrices cannot be written in place");
    }
    average_kernel<<<row_blocks(n), kThreads, 0, (cudaStream_t)stream>>>(m, count, div, n, out);
    return mub::check_launch("snf_average");
}

extern "C" int mub_snf_dominate_f64(const int64_t* ptr, const int32_t* col, const double* val, int64_t n,
                                    double* cs, double* out, mub_stream_t stream) {
    MUB_REQUIRE(n >= 1 && n <= MUB_SNF_MAX_CELLS, "snf: %lld cells", (long long)n);
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned blocks = (unsigned)((n + 255) / 256);
    colsum_kernel<<<blocks, 256, 0, st>>>(ptr, val, n, cs);
    scale_kernel<<<blocks, 256, 0, st>>>(ptr, col, val, n, cs, out);
    return mub::check_launch("snf_dominate");
}

extern "C" int mub_snf_diffuse_f64(const int64_t* s_ptr, const int32_t* s_col, const double* s_val, int64_t n,
                                   const double* B, const double* rB, double* out, int32_t mode,
                                   mub_stream_t stream) {
    MUB_REQUIRE(n >= 1 && n <= MUB_SNF_MAX_CELLS, "snf: %lld cells", (long long)n);
    MUB_REQUIRE(B != out, "snf: the diffusion reads B and writes out; they must not alias");
    const unsigned t = (unsigned)((n + kTile - 1) / kTile);
    cudaStream_t st = (cudaStream_t)stream;
    if (mode == MUB_SNF_DIFFUSE_TRANSPOSED)
        diffuse_kernel<false><<<dim3(t, t), kThreads, 0, st>>>(s_ptr, s_col, s_val, n, B, rB, out);
    else if (mode == MUB_SNF_DIFFUSE_SYMMETRIC)
        diffuse_kernel<true><<<dim3(t, t), kThreads, 0, st>>>(s_ptr, s_col, s_val, n, B, rB, out);
    else
        MUB_REQUIRE(false, "snf: diffusion mode %d", mode);
    return mub::check_launch("snf_diffuse");
}
