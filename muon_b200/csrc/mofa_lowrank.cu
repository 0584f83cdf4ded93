// MOFA non-gaussian likelihoods on a SPARSE view, without the dense N x D pseudo-data.
//
// mofa_pseudo.cu forms yhat = zeta - sigmoid(zeta) (1 - y / r(zeta)) / kappa_d (poisson) or
// zeta - (sigmoid(zeta) - y) / kappa_d (bernoulli) on a dense matrix.  Every such term splits into a part that
// depends on zeta = Z W^T alone and a correction at the stored non-zeros (an implicit zero has y = 0):
//   yhat = g(zeta) + s,   g = zeta - sigmoid(zeta) / kappa_d,
//   s    = y sigmoid(zeta) / (kappa_d r(zeta))  (poisson),   y / kappa_d  (bernoulli),   r = max(softplus, 1e-30)
//   ln p = -r(zeta) + y ln r(zeta)             (poisson),   -softplus(zeta) + y zeta   (bernoulli)
// g is a function of a rank-K matrix, so the contractions with it are evaluated tile by tile and never stored:
//   lowrank_sweep_kernel : a CTA owns 64 rows of one factor matrix and streams 64-row tiles of the other; it forms
//                          the 64 x 64 tile of zeta in registers (4 x 4 per thread, fp32 FMA), applies g, and
//                          contracts the tile with an operand indexed by the streamed rows (out = g C), the
//                          output accumulated on chip and written once.  Without an operand it sums ln p instead.
//   lowrank_nnz_kernel   : the corrections, one warp per row of a CSR (cells) or of a transposed pairs panel
//                          (features); zeta at each stored entry is the dot product of the two factor rows,
//                          formed by the lane that holds the entry.
// Formulas and clamps are those of mofa_pseudo.cu (fp32; 1/kappa is applied as a product).
#include <math.h>

#include "common.cuh"

namespace mub {
namespace {

constexpr int kTile = 64;          // owned and streamed rows per tile of the sweep
constexpr int kSweepThreads = 256;  // 16 x 16 threads, 4 x 4 elements of the zeta tile each

__device__ __forceinline__ float lr_softplus(float z) { return z > 20.f ? z : log1pf(__expf(z)); }
__device__ __forceinline__ float lr_sigmoid(float z) { return __frcp_rn(1.f + __expf(-z)); }
__device__ __forceinline__ float lr_rate(float z) { return fmaxf(lr_softplus(z), 1e-30f); }

// rows [r0, r0 + kTile) of X[nr x LD] into S[LD][kTile] (k-major), rows past nr as zeros
template <int LD>
__device__ __forceinline__ void load_kmajor(const float* __restrict__ X, int64_t r0, int64_t nr, float* S, int tid) {
    for (int i = tid; i < kTile * LD / 4; i += kSweepThreads) {
        const int r = i / (LD / 4), k = (i % (LD / 4)) * 4;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (r0 + r < nr) v = ld_gather4(X + (r0 + r) * LD + k);
        S[(k + 0) * kTile + r] = v.x;
        S[(k + 1) * kTile + r] = v.y;
        S[(k + 2) * kTile + r] = v.z;
        S[(k + 3) * kTile + r] = v.w;
    }
}

// rows [r0, r0 + kTile) of X[nr x LD] into S[kTile][LD] (row-major), rows past nr as zeros
template <int LD>
__device__ __forceinline__ void load_rows(const float* __restrict__ X, int64_t r0, int64_t nr, float* S, int tid) {
    for (int i = tid; i < kTile * LD / 4; i += kSweepThreads) {
        const int r = i / (LD / 4), k = (i % (LD / 4)) * 4;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (r0 + r < nr) v = ld_gather4(X + (r0 + r) * LD + k);
        *reinterpret_cast<float4*>(S + r * LD + k) = v;
    }
}

__device__ __forceinline__ void block_add_double(double v, double* out) {
    __shared__ double part[kSweepThreads / 32];
    v = warp_sum(v);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0) part[w] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int j = 0; j < kSweepThreads / 32; ++j) s += part[j];
        atomicAdd(out, s);
    }
}

// Owned rows A[na x LD], streamed rows Bs[nb x LD], zeta_ab = A_a . B_b.
//   LOGLIK = false: O[a] (=|+=) sum_b g(zeta_ab) C[b] for C[nb x LD];  COLS: kappa is indexed by a (owned rows are
//                   features) and ssq[a] = sum_b g^2 (fp64) is written; else kappa is indexed by b.
//   LOGLIK = true : *ll += sum_ab -r(zeta) (poisson) / -softplus(zeta) (bernoulli), fp64 per CTA.
template <int LD, bool COLS, bool LOGLIK>
__global__ void __launch_bounds__(kSweepThreads)
lowrank_sweep_kernel(const float* __restrict__ A, int64_t na, const float* __restrict__ B, int64_t nb,
                     const float* __restrict__ C, const float* __restrict__ kappa, int32_t kind, float* __restrict__ O,
                     int32_t accumulate, double* __restrict__ ssq, double* __restrict__ ll) {
    constexpr int CW = LD / 16;                           // output columns per thread
    extern __shared__ __align__(16) float smem[];
    float* As = smem;                                     // [LD][kTile]
    float* Bs = As + LD * kTile;                          // [LD][kTile]
    float* Cs = Bs + LD * kTile;                          // [kTile][LD]
    float* Gs = Cs + kTile * LD;                          // [kTile][kTile], owned-major
    const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
    const int64_t a0 = (int64_t)blockIdx.x * kTile;
    load_kmajor<LD>(A, a0, na, As, tid);
    float inv_ka[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int64_t a = a0 + ty * 4 + i;
        inv_ka[i] = (COLS && !LOGLIK && a < na) ? __frcp_rn(__ldg(kappa + a)) : 0.f;
    }
    float o[4][CW];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int c = 0; c < CW; ++c) o[i][c] = 0.f;
    double sq[4] = {0.0, 0.0, 0.0, 0.0};
    double lsum = 0.0;

    for (int64_t b0 = 0; b0 < nb; b0 += kTile) {
        load_kmajor<LD>(B, b0, nb, Bs, tid);
        if (!LOGLIK) load_rows<LD>(C, b0, nb, Cs, tid);
        __syncthreads();
        float z[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) z[i][j] = 0.f;
#pragma unroll 8
        for (int k = 0; k < LD; ++k) {
            const float4 av = *reinterpret_cast<const float4*>(As + k * kTile + ty * 4);
            const float4 bv = *reinterpret_cast<const float4*>(Bs + k * kTile + tx * 4);
            const float a4[4] = {av.x, av.y, av.z, av.w}, b4[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) z[i][j] = fmaf(a4[i], b4[j], z[i][j]);
        }
        bool bval[4];
        float inv_kb[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int64_t b = b0 + tx * 4 + j;
            bval[j] = b < nb;
            inv_kb[j] = (!COLS && !LOGLIK && bval[j]) ? __frcp_rn(__ldg(kappa + b)) : 0.f;
        }
        if (LOGLIK) {
            float part = 0.f;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                if (a0 + ty * 4 + i >= na) continue;
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (bval[j]) part -= kind == 1 ? lr_rate(z[i][j]) : lr_softplus(z[i][j]);
            }
            lsum += (double)part;
        } else {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                float g[4], part = 0.f;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float ik = COLS ? inv_ka[i] : inv_kb[j];
                    g[j] = bval[j] ? z[i][j] - lr_sigmoid(z[i][j]) * ik : 0.f;
                    part = fmaf(g[j], g[j], part);
                }
                if (COLS) sq[i] += (double)part;
                *reinterpret_cast<float4*>(Gs + (ty * 4 + i) * kTile + tx * 4) = make_float4(g[0], g[1], g[2], g[3]);
            }
            __syncthreads();
#pragma unroll 2
            for (int b = 0; b < kTile; b += 4) {
                float gv[4][4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float4 t = *reinterpret_cast<const float4*>(Gs + (ty * 4 + i) * kTile + b);
                    gv[i][0] = t.x, gv[i][1] = t.y, gv[i][2] = t.z, gv[i][3] = t.w;
                }
#pragma unroll
                for (int bb = 0; bb < 4; ++bb) {
                    float cv[CW];
                    const float* cr = Cs + (b + bb) * LD + tx * CW;
                    if constexpr (CW == 4) {
                        const float4 t = *reinterpret_cast<const float4*>(cr);
                        cv[0] = t.x, cv[1] = t.y, cv[2] = t.z, cv[3] = t.w;
                    } else {
                        const float2 t = *reinterpret_cast<const float2*>(cr);
                        cv[0] = t.x, cv[1] = t.y;
                    }
#pragma unroll
                    for (int i = 0; i < 4; ++i)
#pragma unroll
                        for (int c = 0; c < CW; ++c) o[i][c] = fmaf(gv[i][bb], cv[c], o[i][c]);
                }
            }
        }
        __syncthreads();
    }

    if constexpr (LOGLIK) {
        block_add_double(lsum, ll);
    } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int64_t a = a0 + ty * 4 + i;
            if (COLS) {
                double v = sq[i];
#pragma unroll
                for (int off = 8; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
                if (tx == 0 && a < na) ssq[a] = v;
            }
            if (a >= na) continue;
            float* dst = O + a * LD + tx * CW;
#pragma unroll
            for (int c = 0; c < CW; ++c) dst[c] = accumulate ? dst[c] + o[i][c] : o[i][c];
        }
    }
}

// One warp per owned row of a CSR (COLS = false: cells, index = feature) or of a transposed pairs panel (COLS: features,
// index = panel-local cell).  zeta = U[row] . V[index].  With C: O[row] += sum s C[index], and for COLS ssq[row] +=
// sum (2 g s + s^2); without C: *ll += sum y ln r(zeta) (poisson) / y zeta (bernoulli).
template <int LD, bool COLS>
__global__ void __launch_bounds__(256)
lowrank_nnz_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                   const float* __restrict__ values, const int2* __restrict__ pairs, int64_t n_rows,
                   const float* __restrict__ U, const float* __restrict__ V, const float* __restrict__ C,
                   const float* __restrict__ kappa, int32_t kind, float* __restrict__ O, double* __restrict__ ssq,
                   double* __restrict__ ll) {
    constexpr int PL = LD / 32;                           // output columns per lane
    __shared__ __align__(16) float us[8][LD];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int64_t row = (int64_t)blockIdx.x * 8 + w;
    double part = 0.0;
    if (row < n_rows) {                                   // warp-uniform
#pragma unroll
        for (int c = 0; c < PL; ++c) us[w][lane * PL + c] = U[row * LD + lane * PL + c];
        __syncwarp();
        const float ik_row = (COLS && C) ? __frcp_rn(__ldg(kappa + row)) : 0.f;
        float acc[PL];
#pragma unroll
        for (int c = 0; c < PL; ++c) acc[c] = 0.f;
        const int64_t beg = indptr[row], end = indptr[row + 1];
        for (int64_t e0 = beg; e0 < end; e0 += 32) {
            const int64_t e = e0 + lane;
            int idx = 0;
            float s = 0.f;
            if (e < end) {
                float y;
                if (COLS) {
                    const int2 p = ld_stream2(pairs + e);
                    idx = p.x, y = __int_as_float(p.y);
                } else {
                    idx = ld_stream(indices + e), y = ld_stream(values + e);
                }
                const float* vr = V + (int64_t)idx * LD;
                float z = 0.f;
#pragma unroll
                for (int k = 0; k < LD; k += 4) {
                    const float4 v = ld_gather4(vr + k);
                    const float4 u = *reinterpret_cast<const float4*>(&us[w][k]);
                    z = fmaf(u.x, v.x, z), z = fmaf(u.y, v.y, z), z = fmaf(u.z, v.z, z), z = fmaf(u.w, v.w, z);
                }
                if (!C) {
                    part += (double)(kind == 1 ? y * logf(lr_rate(z)) : y * z);
                } else {
                    const float ik = COLS ? ik_row : __frcp_rn(__ldg(kappa + idx));
                    const float sg = lr_sigmoid(z);
                    s = kind == 1 ? y * sg * ik / lr_rate(z) : y * ik;
                    if (COLS) {
                        const float g = z - sg * ik;
                        part += (double)fmaf(2.f * g, s, s * s);
                    }
                }
            }
            if (C) {
                const int cnt = (int)(end - e0 < 32 ? end - e0 : 32);
                for (int j = 0; j < cnt; ++j) {
                    const float sj = __shfl_sync(0xffffffffu, s, j);
                    const int ij = __shfl_sync(0xffffffffu, idx, j);
                    const float* cr = C + (int64_t)ij * LD + lane * PL;
                    if constexpr (PL == 2) {
                        const float2 t = *reinterpret_cast<const float2*>(cr);
                        acc[0] = fmaf(sj, t.x, acc[0]);
                        acc[1] = fmaf(sj, t.y, acc[1]);
                    } else {
                        acc[0] = fmaf(sj, __ldg(cr), acc[0]);
                    }
                }
            }
        }
        if (C) {
#pragma unroll
            for (int c = 0; c < PL; ++c) O[row * LD + lane * PL + c] += acc[c];
            if (COLS) {
                part = warp_sum(part);
                if (lane == 0) ssq[row] += part;
            }
        }
    }
    if (!C) block_add_double(part, ll);
}

template <int LD, bool COLS, bool LOGLIK>
int launch_sweep(const float* A, int64_t na, const float* B, int64_t nb, const float* C, const float* kappa,
                 int32_t kind, float* O, int32_t accumulate, double* ssq, double* ll, cudaStream_t st) {
    const size_t smem = sizeof(float) * (LOGLIK ? 2 * LD * kTile : 3 * LD * kTile + kTile * kTile);
    auto kern = lowrank_sweep_kernel<LD, COLS, LOGLIK>;
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    kern<<<(unsigned)((na + kTile - 1) / kTile), kSweepThreads, smem, st>>>(A, na, B, nb, C, kappa, kind, O, accumulate,
                                                                           ssq, ll);
    return check_launch("mofa_lowrank");
}

template <int LD, bool COLS>
int launch_nnz(const int64_t* indptr, const int32_t* indices, const float* values, const int2* pairs, int64_t n_rows,
               const float* U, const float* V, const float* C, const float* kappa, int32_t kind, float* O,
               double* ssq, double* ll, cudaStream_t st) {
    lowrank_nnz_kernel<LD, COLS><<<(unsigned)((n_rows + 7) / 8), 256, 0, st>>>(indptr, indices, values, pairs, n_rows,
                                                                               U, V, C, kappa, kind, O, ssq, ll);
    return check_launch("mofa_nnz");
}

}  // namespace
}  // namespace mub

#define MUB_LOWRANK_ARGS(ld, kind)                                                               \
    MUB_REQUIRE((ld) == 32 || (ld) == 64, "mofa lowrank: ld must be 32 or 64 (got %d)", (int)(ld)); \
    MUB_REQUIRE((kind) == 1 || (kind) == 2, "mofa lowrank: kind must be 1 (poisson) or 2 (bernoulli)")

extern "C" {

int mub_mofa_lowrank_rows_f32(const float* Z, int64_t n, const float* W, int64_t D, const float* kappa, const float* B,
                              int32_t ld, int32_t kind, float* out, int32_t accumulate, double* loglik,
                              mub_stream_t stream) {
    MUB_LOWRANK_ARGS(ld, kind);
    MUB_REQUIRE(n >= 0 && D >= 0, "mofa_lowrank_rows: negative shape");
    if (n == 0 || D == 0) return 0;
    MUB_REQUIRE(Z && W, "mofa_lowrank_rows: null factor");
    MUB_REQUIRE(B ? (kappa && out) : (loglik != nullptr), "mofa_lowrank_rows: B needs kappa and out, no B needs loglik");
    cudaStream_t st = (cudaStream_t)stream;
    if (!B)
        return ld == 32 ? mub::launch_sweep<32, false, true>(Z, n, W, D, nullptr, nullptr, kind, nullptr, 0, nullptr, loglik, st)
                        : mub::launch_sweep<64, false, true>(Z, n, W, D, nullptr, nullptr, kind, nullptr, 0, nullptr, loglik, st);
    return ld == 32 ? mub::launch_sweep<32, false, false>(Z, n, W, D, B, kappa, kind, out, accumulate, nullptr, nullptr, st)
                    : mub::launch_sweep<64, false, false>(Z, n, W, D, B, kappa, kind, out, accumulate, nullptr, nullptr, st);
}

int mub_mofa_lowrank_cols_f32(const float* Z, int64_t n, const float* W, int64_t D, const float* kappa, const float* C,
                              int32_t ld, int32_t kind, float* P, double* ssq, mub_stream_t stream) {
    MUB_LOWRANK_ARGS(ld, kind);
    MUB_REQUIRE(n >= 0 && D >= 0, "mofa_lowrank_cols: negative shape");
    if (n == 0 || D == 0) return 0;
    MUB_REQUIRE(Z && W && kappa && C && P && ssq, "mofa_lowrank_cols: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    return ld == 32 ? mub::launch_sweep<32, true, false>(W, D, Z, n, C, kappa, kind, P, 0, ssq, nullptr, st)
                    : mub::launch_sweep<64, true, false>(W, D, Z, n, C, kappa, kind, P, 0, ssq, nullptr, st);
}

int mub_mofa_nnz_rows_f32(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_rows,
                          const float* Z, const float* W, const float* kappa, const float* B, int32_t ld, int32_t kind,
                          float* out, double* loglik, mub_stream_t stream) {
    MUB_LOWRANK_ARGS(ld, kind);
    MUB_REQUIRE(n_rows >= 0, "mofa_nnz_rows: negative shape");
    if (n_rows == 0) return 0;
    MUB_REQUIRE(indptr && indices && data && Z && W, "mofa_nnz_rows: null pointer");
    MUB_REQUIRE(B ? (kappa && out) : (loglik != nullptr), "mofa_nnz_rows: B needs kappa and out, no B needs loglik");
    cudaStream_t st = (cudaStream_t)stream;
    return ld == 32 ? mub::launch_nnz<32, false>(indptr, indices, data, nullptr, n_rows, Z, W, B, kappa, kind, out, nullptr, loglik, st)
                    : mub::launch_nnz<64, false>(indptr, indices, data, nullptr, n_rows, Z, W, B, kappa, kind, out, nullptr, loglik, st);
}

int mub_mofa_nnz_cols_f32(const int64_t* t_indptr, const int32_t* t_pairs, int64_t D, const float* Z, const float* W,
                          const float* kappa, const float* C, int32_t ld, int32_t kind, float* P, double* ssq,
                          mub_stream_t stream) {
    MUB_LOWRANK_ARGS(ld, kind);
    MUB_REQUIRE(D >= 0, "mofa_nnz_cols: negative shape");
    if (D == 0) return 0;
    MUB_REQUIRE(t_indptr && t_pairs && Z && W && kappa && C && P && ssq, "mofa_nnz_cols: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const int2* pr = reinterpret_cast<const int2*>(t_pairs);
    return ld == 32 ? mub::launch_nnz<32, true>(t_indptr, nullptr, nullptr, pr, D, W, Z, C, kappa, kind, P, ssq, nullptr, st)
                    : mub::launch_nnz<64, true>(t_indptr, nullptr, nullptr, pr, D, W, Z, C, kappa, kind, P, ssq, nullptr, st);
}

}  // extern "C"
