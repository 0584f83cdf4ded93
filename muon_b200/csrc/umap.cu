// K9 -- UMAP layout: one Jacobi epoch of umap-learn's SGD (optimize_layout_euclidean) per launch.
//
//   Each vertex i is owned by a group of kGroup lanes.  The group reads positions from Y_in and sums, in a fixed
//   order, the clipped gradient terms of
//     - its head entries (CSR row i) sampled this epoch: attraction towards the tail j, then the entry's negative
//       samples k = Philox4x32-10(key, ctr(entry, epoch, draw)) mod n (repulsion, k == i skipped);
//     - its tail entries (row i of the transposed CSR) sampled this epoch: the same attraction from the other end
//       (umap's move_other).
//   Lane l of the group takes the entries l, l + kGroup, ... of each row; the lanes' partial sums are combined by a
//   fixed xor butterfly.  Then Y_out[i] = Y_in[i] + alpha_n * sum.  No atomics, and the sum order depends on the
//   input only, so the layout is bit-identical from run to run.
//
//   Sampling schedule in closed form from eps_e = w_max / w_e >= 1 (no per-entry state): entry e is sampled at
//   epoch n iff floor(n / eps) > floor((n - 1) / eps), i.e. once for each multiple m*eps in (n-1, n].  Its m-th
//   sample draws C(n) - C(n_prev) negatives, with C(x) = floor(x * rate / eps) - 1, n_prev = ceil((m-1) * eps) the
//   epoch of sample m-1 and C = 0 before the first sample.  This is umap's counter arithmetic
//   (epoch_of_next_sample += eps, epoch_of_next_negative_sample += n_neg * eps / rate) carried out exactly: eps is a
//   float32, so every product and quotient below is exact or correctly rounded away from integers in fp64, whereas
//   umap accumulates the counters in fp64 and can land one epoch early or late on a boundary.
#include <math.h>

#include "common.cuh"

namespace mub {
namespace umap {

constexpr int kGroup = 8;     // lanes per vertex (rows of a kNN graph hold ~15-40 entries per side)
constexpr int kThreads = 256;
constexpr float kClip = 4.0f;

// ---- Philox4x32-10 (Salmon et al., SC'11), the same rounds and constants as Random123 / cuRAND -------------------
__host__ __device__ __forceinline__ uint32_t mulhilo(uint32_t a, uint32_t b, uint32_t* hi) {
    const uint64_t p = (uint64_t)a * (uint64_t)b;
    *hi = (uint32_t)(p >> 32);
    return (uint32_t)p;
}

__host__ __device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r > 0) {
            k.x += 0x9E3779B9u;
            k.y += 0xBB67AE85u;
        }
        uint32_t hi0, hi1;
        const uint32_t lo0 = mulhilo(0xD2511F53u, c.x, &hi0);
        const uint32_t lo1 = mulhilo(0xCD9E8D57u, c.z, &hi1);
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    }
    return c;
}

// counter of negative draw `draw` of entry `e` at epoch `epoch`; key = (s0, s1), s2 folded into the counter
__device__ __forceinline__ uint32_t negative_sample(int64_t e, int epoch, int draw, uint32_t s0, uint32_t s1,
                                                    uint32_t s2, uint32_t n) {
    const uint4 ctr = make_uint4((uint32_t)e, (uint32_t)((uint64_t)e >> 32) ^ s2, (uint32_t)epoch, (uint32_t)draw);
    return philox4x32_10(ctr, make_uint2(s0, s1)).x % n;
}

__device__ __forceinline__ bool sampled(int epoch, float eps_f, int* m_out) {
    const double eps = (double)eps_f;
    const int m = (int)floor((double)epoch / eps);
    *m_out = m;
    return epoch >= 1 && m > (int)floor((double)(epoch - 1) / eps);
}

__device__ __forceinline__ int negatives(int epoch, int m, float eps_f, int rate) {
    if (rate <= 0) return 0;
    const double eps = (double)eps_f;
    const int c_now = (int)floor((double)epoch * (double)rate / eps) - 1;
    int c_prev = 0;
    if (m >= 2) {
        const double n_prev = ceil((double)(m - 1) * eps);
        c_prev = (int)floor(n_prev * (double)rate / eps) - 1;
    }
    return max(c_now - c_prev, 0);
}

__device__ __forceinline__ float clip4(float v) { return fminf(kClip, fmaxf(-kClip, v)); }

template <int D>
__device__ __forceinline__ float sqdist(const float* yi, const float* __restrict__ Y, int64_t j, int dim,
                                        float* diff) {
    float d2 = 0.f;
#pragma unroll
    for (int d = 0; d < D; ++d) {
        if (d < dim) {
            diff[d] = yi[d] - __ldg(Y + j * dim + d);
            d2 += diff[d] * diff[d];
        }
    }
    return d2;
}

template <int D>
__device__ __forceinline__ void attract(const float* yi, const float* __restrict__ Y, int64_t j, int dim, float a,
                                        float b, float* acc) {
    float diff[D];
    const float d2 = sqdist<D>(yi, Y, j, dim, diff);
    float gc = 0.f;
    if (d2 > 0.f) {
        const float p = powf(d2, b);
        gc = -2.f * a * b * (p / d2) / (a * p + 1.f);
    }
#pragma unroll
    for (int d = 0; d < D; ++d)
        if (d < dim) acc[d] += clip4(gc * diff[d]);
}

template <int D>
__global__ void __launch_bounds__(kThreads)
epoch_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices, const float* __restrict__ eps,
             const int64_t* __restrict__ t_indptr, const int32_t* __restrict__ t_indices,
             const float* __restrict__ t_eps, int64_t n, int dim, const float* __restrict__ Y,
             float* __restrict__ Y_out, float a, float b, float gamma, float alpha_n, int epoch, int rate,
             uint32_t s0, uint32_t s1, uint32_t s2) {
    const int64_t i = ((int64_t)blockIdx.x * kThreads + threadIdx.x) / kGroup;
    const int lane = threadIdx.x % kGroup;
    const bool live = i < n;   // groups past the end stay for the butterfly (every lane of the warp takes part)
    float yi[D], acc[D];
#pragma unroll
    for (int d = 0; d < D; ++d) {
        yi[d] = live && d < dim ? __ldg(Y + i * dim + d) : 0.f;
        acc[d] = 0.f;
    }
    const int64_t h0 = live ? indptr[i] : 0, h1 = live ? indptr[i + 1] : 0;
    const int64_t t0 = live ? t_indptr[i] : 0, t1 = live ? t_indptr[i + 1] : 0;
    // head side: attraction and negative samples
    for (int64_t e = h0 + lane; e < h1; e += kGroup) {
        const float w = __ldg(eps + e);
        int m;
        if (!sampled(epoch, w, &m)) continue;
        attract<D>(yi, Y, __ldg(indices + e), dim, a, b, acc);
        const int n_neg = negatives(epoch, m, w, rate);
        for (int q = 0; q < n_neg; ++q) {
            const int64_t k = negative_sample(e, epoch, q, s0, s1, s2, (uint32_t)n);
            if (k == i) continue;
            float diff[D];
            const float d2 = sqdist<D>(yi, Y, k, dim, diff);
            if (d2 > 0.f) {
                const float gc = 2.f * gamma * b / ((0.001f + d2) * (a * powf(d2, b) + 1.f));
#pragma unroll
                for (int d = 0; d < D; ++d)
                    if (d < dim) acc[d] += clip4(gc * diff[d]);
            } else {
                // coincident with another vertex: umap's fixed push of +4 in every coordinate
#pragma unroll
                for (int d = 0; d < D; ++d)
                    if (d < dim) acc[d] += kClip;
            }
        }
    }
    // tail side: the head's attraction seen from the tail (clip is odd, so the term is clip(gc * (y_i - y_j)))
    for (int64_t e = t0 + lane; e < t1; e += kGroup) {
        int m;
        if (!sampled(epoch, __ldg(t_eps + e), &m)) continue;
        attract<D>(yi, Y, __ldg(t_indices + e), dim, a, b, acc);
    }
#pragma unroll
    for (int d = 0; d < D; ++d) {
#pragma unroll
        for (int o = kGroup / 2; o > 0; o >>= 1) acc[d] += __shfl_xor_sync(0xffffffffu, acc[d], o, kGroup);
    }
    if (!live) return;
#pragma unroll
    for (int d = 0; d < D; ++d)     // every lane holds the whole sum; lane l writes coordinates l, l + kGroup
        if (d < dim && d % kGroup == lane) Y_out[i * dim + d] = yi[d] + alpha_n * acc[d];
}

__global__ void philox_kernel(const uint32_t* __restrict__ ctr, int64_t n, uint32_t k0, uint32_t k1,
                              uint32_t* __restrict__ out) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const uint4 r = philox4x32_10(make_uint4(ctr[4 * t], ctr[4 * t + 1], ctr[4 * t + 2], ctr[4 * t + 3]),
                                  make_uint2(k0, k1));
    out[4 * t] = r.x;
    out[4 * t + 1] = r.y;
    out[4 * t + 2] = r.z;
    out[4 * t + 3] = r.w;
}

}  // namespace umap
}  // namespace mub

using namespace mub::umap;

extern "C" int mub_umap_epoch_f32(const int64_t* indptr, const int32_t* indices, const float* eps,
                                  const int64_t* t_indptr, const int32_t* t_indices, const float* t_eps, int64_t n,
                                  int32_t dim, const float* Y_in, float* Y_out, float a, float b, float gamma,
                                  float alpha_n, int32_t epoch, int32_t negative_sample_rate, uint32_t s0,
                                  uint32_t s1, uint32_t s2, mub_stream_t stream) {
    MUB_REQUIRE(dim >= 1 && dim <= MUB_UMAP_MAX_COMPONENTS, "umap: n_components %d outside [1, %d]", dim,
                MUB_UMAP_MAX_COMPONENTS);
    MUB_REQUIRE(n >= 1 && n <= 0xffffffffLL, "umap: %lld vertices", (long long)n);
    MUB_REQUIRE(Y_in != Y_out, "umap: the epoch reads Y_in and writes Y_out; they must not alias");
    const int64_t blocks = (n * kGroup + kThreads - 1) / kThreads;
    cudaStream_t st = (cudaStream_t)stream;
#define MUB_UMAP_LAUNCH(D)                                                                                   \
    epoch_kernel<D><<<(unsigned)blocks, kThreads, 0, st>>>(indptr, indices, eps, t_indptr, t_indices, t_eps, \
                                                           n, dim, Y_in, Y_out, a, b, gamma, alpha_n, epoch,  \
                                                           negative_sample_rate, s0, s1, s2)
    if (dim <= 2)
        MUB_UMAP_LAUNCH(2);
    else if (dim <= 4)
        MUB_UMAP_LAUNCH(4);
    else if (dim <= 8)
        MUB_UMAP_LAUNCH(8);
    else
        MUB_UMAP_LAUNCH(16);
#undef MUB_UMAP_LAUNCH
    return mub::check_launch("umap_epoch");
}

extern "C" int mub_philox4x32_10(const uint32_t* ctr, int64_t n, uint32_t k0, uint32_t k1, uint32_t* out,
                                 mub_stream_t stream) {
    MUB_REQUIRE(n >= 0, "philox: n < 0");
    if (n == 0) return 0;
    philox_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(ctr, n, k0, k1, out);
    return mub::check_launch("philox4x32_10");
}
