// K5 -- MOFA+ coordinate-ascent row updates for sm_90a (gaussian views, spike-and-slab weights).
//
// The reference hands densified modalities to mofapy2 (muon/_core/tools.py:117-141,583-585),
// whose per-iteration cost is dense N x D_m GEMMs and elementwise N x D_m passes.  Here the data
// stay sparse and un-centred: the only passes over a modality are two SpMMs per iteration
// (P = Y^T E[Z], Q = Y (tau * E[W]), spmm.cu); centring enters as rank-1 corrections
// (P - mu zsum^T, Q - 1 qshift^T, SURVEY App. C.3) applied on the fly inside these kernels.
//
// What is left are per-row Gauss-Seidel sweeps over the K factors -- sequential in k, independent
// across rows -- so one thread owns one row (feature d for W/Tau, cell n for Z), the K x K moment
// matrix sits in shared memory, and the arithmetic runs in fp64 (K^2 flops per row: negligible
// against the SpMMs) on fp32 storage.  Equations: oracle/mofa_ref.py (update_W, update_Z, tau_b).
#include <math.h>

#include "common.cuh"

namespace mub {

constexpr int kMofaThreads = 128;
constexpr int kMofaKMax = 64;

// ---- W: spike-and-slab weights of one view; G groups of cells with their own tau / means ------------
// Praw[G][D x ld], mu[G][D] (or NULL), zsum[G][K], inv_scale[G], ZZ[G][K x K], tau[G][D]
__global__ void __launch_bounds__(kMofaThreads)
mofa_update_w_kernel(const float* __restrict__ Praw, const float* __restrict__ mu, const double* __restrict__ zsum,
                     const double* __restrict__ inv_scale, const double* __restrict__ ZZ,
                     const float* __restrict__ tau, const double* __restrict__ alpha,
                     const double* __restrict__ lnth, const double* __restrict__ ln1mth, float* __restrict__ W,
                     float* __restrict__ WW, float* __restrict__ S, float* __restrict__ What2, int64_t D, int ld,
                     int K, int G, int spikeslab) {
    extern __shared__ double sm[];
    double* zz = sm;                 // G*K*K
    double* zs = zz + G * K * K;     // G*K
    double* al = zs + G * K;         // K
    double* lo = al + K;             // K : lnth - ln1mth + 0.5 ln alpha
    for (int i = threadIdx.x; i < G * K * K; i += blockDim.x) zz[i] = ZZ[i];
    for (int i = threadIdx.x; i < G * K; i += blockDim.x) zs[i] = zsum ? zsum[i] : 0.0;
    for (int i = threadIdx.x; i < K; i += blockDim.x) {
        al[i] = alpha[i];
        lo[i] = lnth[i] - ln1mth[i] + 0.5 * log(alpha[i]);
    }
    __syncthreads();
    const int64_t d = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= D) return;
    double w[kMofaKMax];
    const size_t off = (size_t)d * ld;
    for (int k = 0; k < K; ++k) w[k] = (double)W[off + k];
    for (int k = 0; k < K; ++k) {
        double a = al[k], b = 0.0;
        for (int g = 0; g < G; ++g) {
            const double* zr = zz + ((size_t)g * K + k) * K;
            const double t_gd = (double)tau[(size_t)g * D + d];
            double cross = 0.0;
            for (int j = 0; j < K; ++j) cross += w[j] * zr[j];
            cross -= w[k] * zr[k];
            const double m_gd = mu ? (double)mu[(size_t)g * D + d] : 0.0;
            const double p = inv_scale[g] * ((double)Praw[(size_t)g * D * ld + off + k] - m_gd * zs[g * K + k]);
            a += t_gd * zr[k];
            b += t_gd * (p - cross);
        }
        const double m = b / a, v = 1.0 / a;
        double s = 1.0;
        if (spikeslab) {
            const double logit = lo[k] - 0.5 * log(a) + 0.5 * b * b / a;
            s = 1.0 / (1.0 + exp(-logit));
        }
        const double m2 = s * (m * m + v);
        w[k] = s * m;
        W[off + k] = (float)w[k];
        WW[off + k] = (float)m2;
        S[off + k] = (float)s;
        What2[off + k] = (float)(m2 + (1.0 - s) / al[k]);
    }
}

// ---- Z: factors; cells fall into C classes (group x set of views they are observed in) ----------------
// qshift[C][K], GW[C][K x K], zvar[C][K]; cls[N] (or NULL = class 0)
__global__ void __launch_bounds__(kMofaThreads)
mofa_update_z_kernel(const float* __restrict__ Q, const double* __restrict__ qshift, const double* __restrict__ GW,
                     const double* __restrict__ zvar, const int32_t* __restrict__ cls, float* __restrict__ Z,
                     int64_t N, int ld, int K, int C) {
    extern __shared__ double sm[];
    double* gw = sm;               // C*K*K
    double* zv = gw + C * K * K;   // C*K
    double* qs = zv + C * K;       // C*K
    for (int i = threadIdx.x; i < C * K * K; i += blockDim.x) gw[i] = GW[i];
    for (int i = threadIdx.x; i < C * K; i += blockDim.x) {
        zv[i] = zvar[i];
        qs[i] = qshift ? qshift[i] : 0.0;
    }
    __syncthreads();
    const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const int c = cls ? cls[n] : 0;
    double z[kMofaKMax];
    const size_t off = (size_t)n * ld;
    for (int k = 0; k < K; ++k) z[k] = (double)Z[off + k];
    for (int k = 0; k < K; ++k) {
        const double* gr = gw + ((size_t)c * K + k) * K;
        double cross = 0.0;
        for (int j = 0; j < K; ++j) cross += z[j] * gr[j];
        cross -= z[k] * gr[k];
        z[k] = zv[c * K + k] * ((double)Q[off + k] - qs[c * K + k] - cross);
        Z[off + k] = (float)z[k];
    }
}

// ---- Tau: 1/2 E||y_d - Z w_d||^2 per feature from sufficient statistics ----------------------
__global__ void __launch_bounds__(kMofaThreads)
mofa_tau_kernel(const float* __restrict__ Praw, const float* __restrict__ mu, const double* __restrict__ zsum,
                double inv_scale, const double* __restrict__ ZZ, const double* __restrict__ ssq,
                const float* __restrict__ W, const float* __restrict__ WW, double b0, double* __restrict__ b_out,
                int64_t D, int ld, int K) {
    extern __shared__ double sm[];
    double* zz = sm;
    double* zs = zz + K * K;
    for (int i = threadIdx.x; i < K * K; i += blockDim.x) zz[i] = ZZ[i];
    for (int i = threadIdx.x; i < K; i += blockDim.x) zs[i] = zsum ? zsum[i] : 0.0;
    __syncthreads();
    const int64_t d = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= D) return;
    double w[kMofaKMax];
    const size_t off = (size_t)d * ld;
    const double m_d = mu ? (double)mu[d] : 0.0;
    double lin = 0.0, quad = 0.0;
    for (int k = 0; k < K; ++k) {
        w[k] = (double)W[off + k];
        lin += w[k] * inv_scale * ((double)Praw[off + k] - m_d * zs[k]);
    }
    for (int k = 0; k < K; ++k) {
        const double* zr = zz + k * K;
        double c = 0.0;
        for (int j = 0; j < K; ++j) c += w[j] * zr[j];
        c -= w[k] * zr[k];
        quad += w[k] * c + (double)WW[off + k] * zr[k];
    }
    b_out[d] = b0 + 0.5 * (ssq[d] - 2.0 * lin + quad);
}

}  // namespace mub

extern "C" {

int mub_mofa_update_w_f32(const float* Praw, const float* mu, const double* zsum, const double* inv_scale,
                          const double* ZZ, const float* tau, const double* alpha, const double* lnth,
                          const double* ln1mth, float* W, float* WW, float* S, float* What2, int64_t D,
                          int32_t ld, int32_t K, int32_t G, int32_t spikeslab, mub_stream_t stream) {
    MUB_REQUIRE(K >= 1 && K <= mub::kMofaKMax && K <= ld, "mofa_update_w: need 1 <= K <= min(64, ld)");
    MUB_REQUIRE(G >= 1, "mofa_update_w: need G >= 1");
    if (D <= 0) return 0;
    MUB_REQUIRE(Praw && inv_scale && ZZ && tau && alpha && lnth && ln1mth && W && WW && S && What2,
                "mofa_update_w: null pointer");
    const size_t smem = sizeof(double) * ((size_t)G * K * K + (size_t)G * K + 2 * K);
    MUB_REQUIRE(smem <= 96 * 1024, "mofa_update_w: groups x factors^2 too large for shared memory (%zu B)", smem);
    if (smem > 48 * 1024)
        cudaFuncSetAttribute(mub::mofa_update_w_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const int grid = (int)((D + mub::kMofaThreads - 1) / mub::kMofaThreads);
    mub::mofa_update_w_kernel<<<grid, mub::kMofaThreads, smem, (cudaStream_t)stream>>>(
        Praw, mu, zsum, inv_scale, ZZ, tau, alpha, lnth, ln1mth, W, WW, S, What2, D, ld, K, G, spikeslab);
    return mub::check_launch("mofa_update_w");
}

int mub_mofa_update_z_f32(const float* Q, const double* qshift, const double* GW, const double* zvar,
                          const int32_t* cls, float* Z, int64_t N, int32_t ld, int32_t K, int32_t C,
                          mub_stream_t stream) {
    MUB_REQUIRE(K >= 1 && K <= mub::kMofaKMax && K <= ld, "mofa_update_z: need 1 <= K <= min(64, ld)");
    MUB_REQUIRE(C >= 1, "mofa_update_z: need C >= 1");
    if (N <= 0) return 0;
    MUB_REQUIRE(Q && GW && zvar && Z, "mofa_update_z: null pointer");
    const size_t smem = sizeof(double) * ((size_t)C * K * K + 2 * (size_t)C * K);
    MUB_REQUIRE(smem <= 96 * 1024, "mofa_update_z: classes x factors^2 too large for shared memory (%zu B)", smem);
    if (smem > 48 * 1024)
        cudaFuncSetAttribute(mub::mofa_update_z_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const int grid = (int)((N + mub::kMofaThreads - 1) / mub::kMofaThreads);
    mub::mofa_update_z_kernel<<<grid, mub::kMofaThreads, smem, (cudaStream_t)stream>>>(Q, qshift, GW, zvar, cls, Z,
                                                                                      N, ld, K, C);
    return mub::check_launch("mofa_update_z");
}

int mub_mofa_tau_f32(const float* Praw, const float* mu, const double* zsum, double inv_scale, const double* ZZ,
                     const double* ssq, const float* W, const float* WW, double b0, double* b_out, int64_t D,
                     int32_t ld, int32_t K, mub_stream_t stream) {
    MUB_REQUIRE(K >= 1 && K <= mub::kMofaKMax && K <= ld, "mofa_tau: need 1 <= K <= min(64, ld)");
    if (D <= 0) return 0;
    MUB_REQUIRE(Praw && ZZ && ssq && W && WW && b_out, "mofa_tau: null pointer");
    const size_t smem = sizeof(double) * ((size_t)K * K + K);
    const int grid = (int)((D + mub::kMofaThreads - 1) / mub::kMofaThreads);
    mub::mofa_tau_kernel<<<grid, mub::kMofaThreads, smem, (cudaStream_t)stream>>>(Praw, mu, zsum, inv_scale, ZZ,
                                                                                 ssq, W, WW, b0, b_out, D, ld, K);
    return mub::check_launch("mofa_tau");
}

}  // extern "C"
