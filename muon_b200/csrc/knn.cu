// Exact brute-force k-nearest-neighbour search (Euclidean), fused distance tiles + top-k selection.
//
// Groundwork for the WNN row (SURVEY 8f-f1): muon's multimodal neighbours need, per modality, the
// n_multineighbors+1 = 201 nearest cells of every cell in a 30-50 dimensional embedding
// (reference muon/_core/preproc.py:520-528 calls umap's NN-descent for this; here the search is exact).
//
// One CTA owns a tile of 64 queries.  Candidate points stream through shared memory in tiles of 64; the
// 64 x 64 block of squared distances is produced GEMM-style (4 x 4 register tile per thread from two
// shared-memory panels; sum of squared differences, no |x|^2+|y|^2-2xy cancellation), then each of the 8 warps updates
// the top-k lists of 8 queries: lists live in shared memory as unsorted (distance, index) arrays with a cached
// current maximum; a candidate below the maximum replaces it and the maximum is recomputed by a warp scan.
// Expected insertions per query are ~k ln(n/k), so selection stays a small fraction of the distance work.
// At the end every list is sorted ascending by (distance, index) and the distances are square-rooted.
//
// fp32 SIMT first (distances accurate to fp32 rounding, self-distance exactly 0, ties resolved by index);
// knn_tc.cu adds a tensor-core (wgmma TF32) candidate pass + fp32 re-rank with the same result.
#include <float.h>

#include "common.cuh"

namespace mub {

constexpr int kKnnQ = 64;        // queries per CTA
constexpr int kKnnC = 64;        // candidates per tile
constexpr int kKnnThreads = 256;
constexpr int kKnnDChunk = 32;   // feature dimensions staged per pass

__global__ void __launch_bounds__(kKnnThreads)
knn_l2_kernel(const float* __restrict__ X, const float* __restrict__ Y, int64_t nq, int64_t nc, int d, int ld, int k,
              int32_t* __restrict__ out_idx, float* __restrict__ out_dist) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* qs = reinterpret_cast<float*>(smem_raw);          // [kKnnDChunk][kKnnQ + 4]  (transposed: dim-major)
    float* cs = qs + kKnnDChunk * (kKnnQ + 4);               // [kKnnDChunk][kKnnC + 4]
    float* dt = cs + kKnnDChunk * (kKnnC + 4);               // [kKnnQ][kKnnC + 1] distance tile
    float* hd = dt + kKnnQ * (kKnnC + 1);                    // [kKnnQ][k] list distances
    int32_t* hi = reinterpret_cast<int32_t*>(hd + (size_t)kKnnQ * k);   // [kKnnQ][k] list indices
    float* hmax = reinterpret_cast<float*>(hi + (size_t)kKnnQ * k);     // [kKnnQ] current maximum
    int32_t* hpos = reinterpret_cast<int32_t*>(hmax + kKnnQ);           // [kKnnQ] position of the maximum

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int tq = tid >> 4, tc = tid & 15;                  // 16 x 16 threads, each a 4 x 4 block
    const int64_t q0 = (int64_t)blockIdx.x * kKnnQ;

    for (int i = tid; i < kKnnQ * k; i += kKnnThreads) {
        hd[i] = FLT_MAX;
        hi[i] = -1;
    }
    if (tid < kKnnQ) {
        hmax[tid] = FLT_MAX;
        hpos[tid] = 0;
    }
    __syncthreads();

    for (int64_t c0 = 0; c0 < nc; c0 += kKnnC) {
        float acc[4][4];
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;
        for (int d0 = 0; d0 < d; d0 += kKnnDChunk) {
            // stage a [dims x points] panel of queries and of candidates (zero beyond n / d)
            for (int idx = tid; idx < kKnnDChunk * kKnnQ; idx += kKnnThreads) {
                const int p = idx / kKnnDChunk, dd = idx % kKnnDChunk;   // consecutive threads: consecutive dims
                const int64_t q = q0 + p, c = c0 + p;
                const int dim = d0 + dd;
                qs[dd * (kKnnQ + 4) + p] = (q < nq && dim < d) ? __ldg(X + (size_t)q * ld + dim) : 0.f;
                cs[dd * (kKnnC + 4) + p] = (c < nc && dim < d) ? __ldg(Y + (size_t)c * ld + dim) : 0.f;
            }
            __syncthreads();
#pragma unroll 8
            for (int dd = 0; dd < kKnnDChunk; ++dd) {
                const float4 a = *reinterpret_cast<const float4*>(qs + dd * (kKnnQ + 4) + tq * 4);
                const float4 b = *reinterpret_cast<const float4*>(cs + dd * (kKnnC + 4) + tc * 4);
                const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const float df = av[i] - bv[j];
                        acc[i][j] = fmaf(df, df, acc[i][j]);
                    }
            }
            __syncthreads();
        }
        // squared distances of the tile -> shared memory (invalid candidates get +inf)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int64_t c = c0 + tc * 4 + j;
                dt[(tq * 4 + i) * (kKnnC + 1) + tc * 4 + j] = (c < nc) ? acc[i][j] : FLT_MAX;
            }
        }
        __syncthreads();
        // selection: warp w owns queries [8w, 8w+8)
        for (int qq = 0; qq < 8; ++qq) {
            const int ql = warp * 8 + qq;
            if (q0 + ql >= nq) break;
            float* ld_ = hd + (size_t)ql * k;
            int32_t* li = hi + (size_t)ql * k;
#pragma unroll
            for (int half = 0; half < kKnnC / 32; ++half) {
                const int cl = half * 32 + lane;
                const float v = dt[ql * (kKnnC + 1) + cl];
                const int32_t ci = (int32_t)(c0 + cl);
                // candidates are visited in increasing index order, so "strictly below the maximum" keeps the
                // lowest-index element among equal distances (same tie rule as a stable sort)
                unsigned m = __ballot_sync(0xffffffffu, v < hmax[ql]);
                while (m) {
                    const int src = __ffs(m) - 1;
                    m &= m - 1;
                    const float cv = __shfl_sync(0xffffffffu, v, src);
                    const int32_t cidx = __shfl_sync(0xffffffffu, ci, src);
                    if (cv < hmax[ql]) {              // warp-uniform (shared value)
                        const int pos = hpos[ql];
                        __syncwarp();
                        if (lane == 0) {
                            ld_[pos] = cv;
                            li[pos] = cidx;
                        }
                        __syncwarp();
                        // recompute the maximum (largest distance, largest index among equals)
                        float bm = -1.f;
                        int bp = 0, bi = -1;
                        for (int t = lane; t < k; t += 32) {
                            const float x = ld_[t];
                            const int xi = li[t];
                            if (x > bm || (x == bm && xi > bi)) { bm = x; bp = t; bi = xi; }
                        }
#pragma unroll
                        for (int o = 16; o > 0; o >>= 1) {
                            const float om = __shfl_xor_sync(0xffffffffu, bm, o);
                            const int op = __shfl_xor_sync(0xffffffffu, bp, o);
                            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                            if (om > bm || (om == bm && oi > bi)) { bm = om; bp = op; bi = oi; }
                        }
                        if (lane == 0) {
                            hmax[ql] = bm;
                            hpos[ql] = bp;
                        }
                        __syncwarp();
                    }
                }
            }
        }
        __syncthreads();
    }
    // final: sort each list ascending by (distance, index) with a warp-level selection sort, write out
    for (int qq = 0; qq < 8; ++qq) {
        const int ql = warp * 8 + qq;
        const int64_t q = q0 + ql;
        if (q >= nq) break;
        float* ld_ = hd + (size_t)ql * k;
        int32_t* li = hi + (size_t)ql * k;
        for (int r = 0; r < k; ++r) {
            float bm = FLT_MAX;
            int bp = -1, bi = 0x7fffffff;
            for (int t = lane; t < k; t += 32) {
                const float x = ld_[t];
                const int xi = li[t];
                if (xi >= 0 && (x < bm || (x == bm && xi < bi))) { bm = x; bp = t; bi = xi; }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const float om = __shfl_xor_sync(0xffffffffu, bm, o);
                const int op = __shfl_xor_sync(0xffffffffu, bp, o);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (op >= 0 && (bp < 0 || om < bm || (om == bm && oi < bi))) { bm = om; bp = op; bi = oi; }
            }
            if (lane == 0) {
                if (bp >= 0) {
                    out_idx[(size_t)q * k + r] = bi;
                    out_dist[(size_t)q * k + r] = sqrtf(bm);
                    li[bp] = -1;          // consumed
                } else {                  // fewer than k candidates
                    out_idx[(size_t)q * k + r] = -1;
                    out_dist[(size_t)q * k + r] = INFINITY;
                }
            }
            __syncwarp();
        }
    }
}

static size_t knn_smem_bytes(int k) {
    return sizeof(float) * ((size_t)kKnnDChunk * (kKnnQ + 4) + (size_t)kKnnDChunk * (kKnnC + 4) +
                            (size_t)kKnnQ * (kKnnC + 1) + (size_t)kKnnQ * k * 2 + 2 * kKnnQ);
}

}  // namespace mub

extern "C" {

int mub_knn_l2_f32(const float* X, int64_t nq, const float* Y, int64_t nc, int32_t d, int32_t ld, int32_t k,
                   int32_t* out_idx, float* out_dist, mub_stream_t stream) {
    MUB_REQUIRE(nq >= 0 && nc >= 0 && d >= 1 && ld >= d, "knn_l2: bad shape");
    MUB_REQUIRE(k >= 1 && k <= 320, "knn_l2: need 1 <= k <= 320 (got %d)", k);
    if (nq == 0) return 0;
    MUB_REQUIRE(X && Y && out_idx && out_dist, "knn_l2: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    const size_t smem = mub::knn_smem_bytes(k);
    cudaError_t e = cudaFuncSetAttribute(mub::knn_l2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) {
        mub::set_error("knn_l2: %zu B of shared memory: %s", smem, cudaGetErrorString(e));
        return -2;
    }
    const unsigned grid = (unsigned)((nq + mub::kKnnQ - 1) / mub::kKnnQ);
    mub::knn_l2_kernel<<<grid, mub::kKnnThreads, smem, s>>>(X, Y, nq, nc, d, ld, k, out_idx, out_dist);
    return mub::check_launch("knn_l2");
}

}  // extern "C"
