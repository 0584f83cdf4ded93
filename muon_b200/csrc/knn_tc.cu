// Exact k-nearest-neighbour search, tensor-core candidate pass + fp32 re-rank (wgmma TF32, sm_90a).
//
// Same contract as knn.cu (mub_knn_l2_f32): the k nearest rows of Y for every row of X in Euclidean distance,
// ascending, ties by lower index, distances bit-identical to the SIMT kernel.  The n x n inner-product matrix is
// the one GEMM-shaped operation of the WNN row (reference muon/_core/preproc.py:520-528), so it runs on the
// Hopper tensor cores:
//
//   pass 1  knn_tc_candidates_kernel: one CTA (one warpgroup of 128 threads) owns 128 queries.  Candidate tiles of
//           128 points are written to shared memory in the canonical no-swizzle K-major layout (8-row x 16-byte core
//           matrices, SBO 128 B between 8-row groups, LBO 2048 B between K chunks); the warpgroup issues
//           2 x ceil(d/8) wgmma.mma_async m64n128k8 TF32 instructions (query rows 0-63 and 64-127) that accumulate
//           S = Q C^T in registers, waits for them, and stages S through shared memory so that thread t holds row t;
//           each thread then forms a(q,c) = |c|^2 - 2 S and keeps every candidate with a <= tau_q in a per-query buffer.
//           TF32 truncates the inputs to 10 mantissa bits, so a() carries an error of at most 2^-8 |q||c| -- too
//           coarse for concentrated distance distributions, so for d <= 64 the operands are split 3xTF32
//           (big + small parts along a tripled K axis, see knn_tc_pack_kernel) and the error drops to ~5e-5 |q||c|.
//           The threshold is tau_q = (k-th smallest a seen so far, rounded up) + 2 * bound.  Order statistics
//           move by at most the perturbation, hence no true k-nearest neighbour is ever rejected (DESIGN.md section 9).
//           When a buffer fills up (1024 entries) the warp re-derives tau by bisection on the float keys and drops
//           what no longer qualifies.
//   pass 2  knn_tc_rerank_kernel: warp per query, exact fp32 squared distances of the surviving candidates with the
//           same arithmetic as knn.cu (sequential fmaf over the dimensions), k rounds of (distance, index) minimum
//           extraction.
//
// Operands are packed once per call (knn_tc_pack_kernel) into per-tile blocks that already have the shared-memory
// layout, so that staging a tile is one contiguous, fully coalesced copy (and can become a single 1-D TMA bulk copy).
// Single-stage (load -> MMA -> epilogue in sequence; the CTAs co-resident on an SM overlap each other), plain
// global->shared copies.
#include <float.h>
#include <math.h>

#include "common.cuh"

namespace mub {

constexpr int kTcM = 128;        // queries per CTA tile (two m64 row halves)
constexpr int kTcN = 128;        // candidates per MMA tile (wgmma N)
constexpr int kTcCap = 1024;     // candidate buffer entries per query
constexpr int kTcThreads = 128;  // one warpgroup
constexpr int kTcSLd = kTcN + 1; // row stride (floats) of the staged score tile: thread t reads row t without bank conflicts

__device__ __forceinline__ uint32_t tc_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// wgmma shared-memory matrix descriptor, K-major, no swizzle (layout type 0 in bits 62-63, base offset 0):
// start address, leading-dimension byte offset (between core matrices along K), stride-dimension byte offset
// (between 8-row groups along M / N), all in 16-byte units
__device__ __forceinline__ uint64_t tc_wgmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    return d;
}

// D[64 x 128] (+)= A[64 x 8] . B[128 x 8]^T in TF32, fp32 accumulators in the warpgroup's registers.  Fragment:
// thread t (warp w = t/32, lane l) holds d[4j + 2i + c] = D[16w + l/4 + 8i][8j + 2(l%4) + c].
__device__ __forceinline__ void tc_wgmma_m64n128k8(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
        "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "
        "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
          "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
          "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(accumulate));
}

// scores of one 128 x 128 tile pair, S = Q C^T -> shared memory sS[row * kTcSLd + col].  sS aliases sC: every wgmma of
// the tile has completed (and every thread passed a barrier) before the first score is stored.
__device__ __forceinline__ void tc_scores(const unsigned char* sQ, const unsigned char* sC, float* sS, int Kp, int tid) {
    float acc[2][64];                                           // no initialisation: the first k-step has scale-d = 0
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
    const uint32_t lbo_q = kTcM * 16, lbo_c = kTcN * 16, sbo = 128;
    for (int ks = 0; ks < Kp / 8; ++ks) {                       // k8 = two 16-byte K chunks
        const uint64_t db = tc_wgmma_desc(tc_smem_u32(sC) + (uint32_t)(2 * ks) * lbo_c, lbo_c, sbo);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const uint64_t da = tc_wgmma_desc(tc_smem_u32(sQ) + (uint32_t)(2 * ks) * lbo_q + (uint32_t)h * 64 * 16, lbo_q, sbo);
            tc_wgmma_m64n128k8(acc[h], da, db, ks > 0 ? 1u : 0u);
        }
    }
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
    __syncthreads();
    const int w = tid >> 5, l = tid & 31;
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < kTcN / 8; ++j)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                float* dst = sS + (size_t)(h * 64 + 16 * w + (l >> 2) + 8 * i) * kTcSLd + 8 * j + 2 * (l & 3);
                dst[0] = acc[h][4 * j + 2 * i];
                dst[1] = acc[h][4 * j + 2 * i + 1];
            }
    __syncthreads();
}

// monotone map float -> uint32 (order preserving, total on non-NaN)
__device__ __forceinline__ uint32_t tc_okey(float x) {
    const uint32_t u = __float_as_uint(x);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float tc_from_okey(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

// Pack X[n x ld] into 128-row tiles in the canonical UMMA K-major layout: float4 index (tile*chunks_total + c)*128 + r
// holds 4 consecutive K values of row tile*128+r (zero beyond d and beyond n); also |x|^2 (sequential fmaf) and its
// maximum.  split = 0: K = the Kp padded dimensions.  split = 1 / 2 (query / candidate side): 3xTF32 -- every value
// is written as big = x truncated to TF32 (exactly representable, so the tensor core's own truncation is a no-op) and
// small = x - big (exact in fp32); the K axis is [big | big | small] for queries and [big | small | big] for
// candidates, so that one K = 3 Kp product gives qb.cb + qb.cs + qs.cb = q.c up to ~3 * 2^-20 |q||c|.
__global__ void knn_tc_pack_kernel(const float* __restrict__ X, int64_t n, int d, int ld, int Kp, int split,
                                   float4* __restrict__ pk, float* __restrict__ norms, unsigned int* __restrict__ maxbits) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t n_pad = (n + kTcM - 1) / kTcM * kTcM;
    if (i >= n_pad) return;
    const int64_t tile = i / kTcM;
    const int r = (int)(i % kTcM);
    const int chunks = Kp / 4;
    const int chunks_total = split ? 3 * chunks : chunks;
    const bool live = i < n;
    float s = 0.f;
    for (int c = 0; c < chunks; ++c) {
        float v[4], big[4], small[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int dim = c * 4 + e;
            v[e] = (live && dim < d) ? X[(size_t)i * ld + dim] : 0.f;
            s = fmaf(v[e], v[e], s);
            big[e] = __uint_as_float(__float_as_uint(v[e]) & 0xFFFFE000u);
            small[e] = v[e] - big[e];
        }
        float4* dst = pk + ((size_t)tile * chunks_total + c) * kTcM + r;
        if (!split) {
            *dst = make_float4(v[0], v[1], v[2], v[3]);
        } else {
            const float4 b4 = make_float4(big[0], big[1], big[2], big[3]);
            const float4 s4 = make_float4(small[0], small[1], small[2], small[3]);
            dst[0] = b4;
            dst[(size_t)chunks * kTcM] = (split == 1) ? b4 : s4;
            dst[(size_t)2 * chunks * kTcM] = (split == 1) ? s4 : b4;
        }
    }
    if (live) {
        norms[i] = s;
        if (maxbits) atomicMax(maxbits, __float_as_uint(s));   // s >= 0: the bit pattern is monotone
    }
}

// Re-derive tau from the buffer (k-th smallest key, rounded up to a 2^12-ulp bucket, plus the slack) and drop the
// entries above it.  Called warp-wide; every lane works on its own column of the [cap][128] buffers and of the
// [16][128] shared-memory histogram `hist` (radix select on the 20-bit key prefix, 4 bits per pass).
__device__ __forceinline__ void tc_compact(float* __restrict__ kb, int32_t* __restrict__ ib, int32_t* __restrict__ hist,
                                           int tid, int k, float slack, int& cnt, float& tau) {
    if (cnt >= k) {
        uint32_t H = 0;          // high digits of the k-th smallest prefix found so far
        int below = 0;           // entries whose prefix is below every prefix starting with H
#pragma unroll 1
        for (int s = 16; s >= 0; s -= 4) {
#pragma unroll
            for (int j = 0; j < 16; ++j) hist[j * kTcM + tid] = 0;
            // eight independent buffer loads in flight, then the (dependent, shared-memory) histogram updates: with one
            // load per update the compiler cannot move the loads above the updates (generic pointers may alias) and
            // every element paid a full L2 round trip -- this loop was the whole cost of the candidate pass
            for (int i = 0; i < cnt; i += 8) {
                float v8[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) v8[u] = (i + u < cnt) ? kb[(size_t)(i + u) * kTcM + tid] : 0.f;
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    if (i + u < cnt) {
                        const uint32_t p = tc_okey(v8[u]) >> 12;
                        if ((p >> (s + 4)) == H) hist[((p >> s) & 15u) * kTcM + tid] += 1;
                    }
                }
            }
            int acc = below, D = 15;
            bool found = false;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int hj = hist[j * kTcM + tid];
                if (!found) {
                    if (acc + hj >= k) { D = j; found = true; }
                    else acc += hj;
                }
            }
            below = acc;
            H = (H << 4) | (uint32_t)D;
        }
        float base = tc_from_okey((H << 12) | 0xFFFu);    // upper end of the bucket holding the k-th smallest key
        if (!(base <= FLT_MAX)) base = FLT_MAX;            // bucket top beyond the finite range (or NaN pattern)
        tau = base + slack;
        int w = 0;
        for (int i = 0; i < cnt; i += 8) {                 // same batching: 16 loads in flight, then the in-place writes (w <= i)
            float v8[8];
            int32_t j8[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const bool ok = i + u < cnt;
                v8[u] = ok ? kb[(size_t)(i + u) * kTcM + tid] : 0.f;
                j8[u] = ok ? ib[(size_t)(i + u) * kTcM + tid] : 0;
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                if (i + u < cnt && v8[u] <= tau) {
                    kb[(size_t)w * kTcM + tid] = v8[u];
                    ib[(size_t)w * kTcM + tid] = j8[u];
                    ++w;
                }
            }
        }
        cnt = w;
    }
}

__global__ void __launch_bounds__(kTcThreads)
knn_tc_candidates_kernel(const float4* __restrict__ Xpk, const float* __restrict__ xnorm, int64_t nq,
                         const float4* __restrict__ Ypk, const float* __restrict__ ynorm, int64_t nc, int Kp,
                         int k, float slack_rel, const unsigned int* __restrict__ ymax_bits, float* __restrict__ kbuf,
                         int32_t* __restrict__ ibuf, int32_t* __restrict__ cand, int32_t* __restrict__ cand_cnt,
                         int32_t* __restrict__ status) {
    extern __shared__ __align__(1024) unsigned char smem[];
    const int tid = threadIdx.x;
    const int chunks = Kp / 4;                                  // 16-byte K chunks (4 tf32 values)
    unsigned char* sQ = smem;                                   // [chunks][128][16 B]
    unsigned char* sC = smem + (size_t)chunks * kTcM * 16;      // [chunks][128][16 B], then the score tile in its place
    float* sS = reinterpret_cast<float*>(sC);                   // [128][kTcSLd]
    const size_t c_bytes = (size_t)chunks * kTcN * 16, s_bytes = sizeof(float) * kTcM * kTcSLd;
    float* sCn = reinterpret_cast<float*>(sC + (c_bytes > s_bytes ? c_bytes : s_bytes));   // [2][128] candidate norms
    int32_t* hist = reinterpret_cast<int32_t*>(sCn + 2 * kTcN);               // [16][128] radix-select counters

    float* kb = kbuf + (size_t)blockIdx.x * kTcCap * kTcM;
    int32_t* ib = ibuf + (size_t)blockIdx.x * kTcCap * kTcM;
    const float cmax = sqrtf(__uint_as_float(*ymax_bits));

    const int64_t n_qt = (nq + kTcM - 1) / kTcM;
    uint32_t it = 0;                                            // candidate tiles processed so far (norm buffer = it & 1)
    for (int64_t qt = blockIdx.x; qt < n_qt; qt += gridDim.x) {
        const int64_t row = qt * kTcM + tid;
        const bool live = row < nq;
        __syncthreads();                                        // the previous query tile's wgmma reads of sQ are done
        {   // the packed tile already has the shared-memory layout: contiguous copy
            const float4* src = Xpk + (size_t)qt * chunks * kTcM;
            float4* dst = reinterpret_cast<float4*>(sQ);
#pragma unroll 4
            for (int i = tid; i < chunks * kTcM; i += kTcThreads) dst[i] = __ldg(src + i);
        }
        const float qn = live ? xnorm[row] : 0.f;
        // 2 x (error bound of a(), slack_rel/2 * |q| max|c|: see the host code) plus fp32 rounding of the norms
        const float slack = slack_rel * sqrtf(qn) * cmax + 1e-5f * (qn + cmax * cmax);
        // another CTA already found a query whose error band is too crowded: the caller will use the SIMT kernel
        if (__syncthreads_or(*reinterpret_cast<volatile int32_t*>(status) & 2)) break;   // block-uniform decision
        float tau = live ? INFINITY : -INFINITY;
        int cnt = 0;
        int overflow = 0;

        for (int64_t c0 = 0; c0 < nc; c0 += kTcN, ++it) {
            if (__any_sync(0xffffffffu, cnt > kTcCap - kTcN)) {
                tc_compact(kb, ib, hist, tid, k, slack, cnt, tau);
                if (cnt > kTcCap - kTcN) {                      // more than 896 candidates inside the slack band
                    overflow = 1;
                    cnt = kTcCap - kTcN;
                    atomicOr(status, 2);
                }
            }
            const int64_t crow = c0 + tid;
            const bool cl = crow < nc;
            __syncthreads();                                    // every thread has read the previous score tile (sS = sC)
            {
                const float4* src = Ypk + (size_t)(c0 / kTcN) * chunks * kTcN;
                float4* dst = reinterpret_cast<float4*>(sC);
#pragma unroll 4
                for (int i = tid; i < chunks * kTcN; i += kTcThreads) dst[i] = __ldg(src + i);
            }
            float* cn = sCn + (it & 1) * kTcN;
            cn[tid] = cl ? ynorm[crow] : INFINITY;
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic stores -> async proxy (wgmma reads)
            __syncthreads();
            tc_scores(sQ, sC, sS, Kp, tid);
            const float* srow = sS + (size_t)tid * kTcSLd;
            for (int cc = 0; cc < kTcN; cc += 32) {
#pragma unroll
                for (int j = 0; j < 32; ++j) {
                    const float a = fmaf(-2.f, srow[cc + j], cn[cc + j]);
                    if (a <= tau && c0 + cc + j < nc) {
                        if (cnt < kTcCap) {
                            kb[(size_t)cnt * kTcM + tid] = a;
                            ib[(size_t)cnt * kTcM + tid] = (int32_t)(c0 + cc + j);
                            ++cnt;
                        } else {
                            overflow = 1;
                        }
                    }
                }
            }
        }
        tc_compact(kb, ib, hist, tid, k, slack, cnt, tau);      // final trim
        if (live) {
            cand_cnt[row] = cnt;
            for (int i = 0; i < cnt; ++i) cand[(size_t)row * kTcCap + i] = ib[(size_t)i * kTcM + tid];
            if (overflow) atomicOr(status, 2);
        }
    }
}

constexpr int kTcRerankWarps = 4;

__global__ void __launch_bounds__(kTcRerankWarps * 32)
knn_tc_rerank_kernel(const float* __restrict__ X, int64_t nq, const float* __restrict__ Y, int d, int ld, int k,
                     const int32_t* __restrict__ cand, const int32_t* __restrict__ cand_cnt,
                     int32_t* __restrict__ out_idx, float* __restrict__ out_dist) {
    __shared__ float sd_all[kTcRerankWarps][kTcCap];
    __shared__ int32_t si_all[kTcRerankWarps][kTcCap];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t row = (int64_t)blockIdx.x * kTcRerankWarps + warp;
    if (row >= nq) return;
    float* sd = sd_all[warp];
    int32_t* si = si_all[warp];
    int n = cand_cnt[row];
    n = n < 0 ? 0 : (n > kTcCap ? kTcCap : n);
    const float* xq = X + (size_t)row * ld;
    for (int i = lane; i < n; i += 32) {
        const int32_t j = cand[(size_t)row * kTcCap + i];
        const float* yc = Y + (size_t)j * ld;
        float acc = 0.f;
        for (int t = 0; t < d; ++t) {                           // same arithmetic as knn.cu: sequential fmaf of differences
            const float df = __ldg(xq + t) - __ldg(yc + t);
            acc = fmaf(df, df, acc);
        }
        sd[i] = acc;
        si[i] = j;
    }
    __syncwarp();
    for (int r = 0; r < k; ++r) {
        float bm = FLT_MAX;
        int bp = -1, bi = 0x7fffffff;
        for (int t = lane; t < n; t += 32) {
            const float x = sd[t];
            const int xi = si[t];
            if (xi >= 0 && (bp < 0 || x < bm || (x == bm && xi < bi))) { bm = x; bp = t; bi = xi; }
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
                out_idx[(size_t)row * k + r] = bi;
                out_dist[(size_t)row * k + r] = sqrtf(bm);
                si[bp] = -1;
            } else {
                out_idx[(size_t)row * k + r] = -1;
                out_dist[(size_t)row * k + r] = INFINITY;
            }
        }
        __syncwarp();
    }
}

struct TcLayout {
    size_t xnorm, ynorm, ymax, cnt, cand, kbuf, ibuf, xpk, ypk, total;
    int grid, Kp, Ktot, split;
};

static TcLayout tc_layout(int64_t nq, int64_t nc, int d) {
    auto up = [](size_t x) { return (x + 255) & ~(size_t)255; };
    TcLayout L;
    const int64_t n_qt = (nq + kTcM - 1) / kTcM;
    int g = 2 * sm_count();
    if (g > n_qt) g = (int)(n_qt > 0 ? n_qt : 1);
    L.grid = g;
    size_t o = 0;
    L.xnorm = o; o = up(o + sizeof(float) * (size_t)nq);
    L.ynorm = o; o = up(o + sizeof(float) * (size_t)nc);
    L.ymax = o;  o = up(o + 256);
    L.cnt = o;   o = up(o + sizeof(int32_t) * (size_t)nq);
    L.cand = o;  o = up(o + sizeof(int32_t) * (size_t)nq * kTcCap);
    L.kbuf = o;  o = up(o + sizeof(float) * (size_t)g * kTcCap * kTcM);
    L.ibuf = o;  o = up(o + sizeof(int32_t) * (size_t)g * kTcCap * kTcM);
    L.Kp = (d + 7) / 8 * 8;
    L.split = d <= 64 ? 1 : 0;                 // 3xTF32 operands need 3 * Kp * 1 KB of shared memory per tile pair
    L.Ktot = L.split ? 3 * L.Kp : L.Kp;
    L.xpk = o;   o = up(o + sizeof(float) * (size_t)((nq + kTcM - 1) / kTcM) * kTcM * L.Ktot);
    L.ypk = o;   o = up(o + sizeof(float) * (size_t)((nc + kTcN - 1) / kTcN) * kTcN * L.Ktot);
    L.total = o;
    return L;
}

}  // namespace mub

extern "C" {

size_t mub_knn_l2_tc_workspace_bytes(int64_t nq, int64_t nc, int32_t d) {
    if (nq < 0 || nc < 0 || d < 1 || d > 128) return 0;
    return mub::tc_layout(nq, nc, d).total;
}

int mub_knn_l2_tc_f32(const float* X, int64_t nq, const float* Y, int64_t nc, int32_t d, int32_t ld, int32_t k,
                      int32_t* out_idx, float* out_dist, void* workspace, size_t workspace_bytes, int32_t* status,
                      mub_stream_t stream) {
    MUB_REQUIRE(nq >= 0 && nc >= 0 && d >= 1 && ld >= d, "knn_l2_tc: bad shape");
    MUB_REQUIRE(d <= 128, "knn_l2_tc: d <= 128 (got %d)", d);
    MUB_REQUIRE(k >= 1 && k <= 512, "knn_l2_tc: need 1 <= k <= 512 (got %d)", k);
    MUB_REQUIRE(nc < (int64_t)1 << 31, "knn_l2_tc: more than 2^31 candidates");
    if (nq == 0) return 0;
    MUB_REQUIRE(X && Y && out_idx && out_dist && workspace && status, "knn_l2_tc: null pointer");
    const mub::TcLayout L = mub::tc_layout(nq, nc, d);
    MUB_REQUIRE(workspace_bytes >= L.total, "knn_l2_tc: workspace of %zu B, need %zu B", workspace_bytes, L.total);
    cudaStream_t s = (cudaStream_t)stream;
    unsigned char* ws = (unsigned char*)workspace;
    float* xnorm = (float*)(ws + L.xnorm);
    float* ynorm = (float*)(ws + L.ynorm);
    unsigned int* ymax = (unsigned int*)(ws + L.ymax);
    int32_t* cnt = (int32_t*)(ws + L.cnt);
    int32_t* cand = (int32_t*)(ws + L.cand);
    float* kbuf = (float*)(ws + L.kbuf);
    int32_t* ibuf = (int32_t*)(ws + L.ibuf);
    cudaError_t e = cudaMemsetAsync(ymax, 0, 4, s);
    if (e != cudaSuccess) {
        mub::set_error("knn_l2_tc: memset: %s", cudaGetErrorString(e));
        return -2;
    }
    float4* xpk = (float4*)(ws + L.xpk);
    float4* ypk = (float4*)(ws + L.ypk);
    const int Kp = L.Kp, Ktot = L.Ktot;
    const int64_t nq_pad = (nq + mub::kTcM - 1) / mub::kTcM * mub::kTcM, nc_pad = (nc + mub::kTcN - 1) / mub::kTcN * mub::kTcN;
    mub::knn_tc_pack_kernel<<<(unsigned)(nq_pad / 128), 128, 0, s>>>(X, nq, d, ld, Kp, L.split ? 1 : 0, xpk, xnorm, nullptr);
    if (nc > 0)
        mub::knn_tc_pack_kernel<<<(unsigned)(nc_pad / 128), 128, 0, s>>>(Y, nc, d, ld, Kp, L.split ? 2 : 0, ypk, ynorm, ymax);
    // error of a() = |c|^2 - 2 S:  plain TF32 truncates both inputs to 10 mantissa bits -> |dS| <= 2^-9 |q||c|, so
    // |da| <= 2^-8 |q||c|; 3xTF32 leaves ~3 * 2^-20 from the dropped/truncated small parts plus the fp32 accumulation of
    // K <= 192 terms (<= 2^-23 each) -> |da| <= 4.6e-5 |q||c|.  tau needs twice the bound; the plain variant doubles it
    // once more for safety.
    const float slack_rel = L.split ? 1.2e-4f : 4.f * 0.00390625f;
    const size_t c_bytes = (size_t)(Ktot / 4) * mub::kTcN * 16, s_bytes = sizeof(float) * mub::kTcM * mub::kTcSLd;
    const size_t smem = (size_t)(Ktot / 4) * mub::kTcM * 16 + (c_bytes > s_bytes ? c_bytes : s_bytes) +
                        2 * mub::kTcN * sizeof(float) + 16 * mub::kTcM * sizeof(int32_t);
    e = cudaFuncSetAttribute(mub::knn_tc_candidates_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) {
        mub::set_error("knn_l2_tc: %zu B of shared memory: %s", smem, cudaGetErrorString(e));
        return -2;
    }
    mub::knn_tc_candidates_kernel<<<L.grid, mub::kTcThreads, smem, s>>>(xpk, xnorm, nq, ypk, ynorm, nc, Ktot, k, slack_rel, ymax,
                                                                         kbuf, ibuf, cand, cnt, status);
    int rc = mub::check_launch("knn_l2_tc candidates");
    if (rc) return rc;
    mub::knn_tc_rerank_kernel<<<(unsigned)((nq + mub::kTcRerankWarps - 1) / mub::kTcRerankWarps), mub::kTcRerankWarps * 32, 0, s>>>(
        X, nq, Y, d, ld, k, cand, cnt, out_idx, out_dist);
    return mub::check_launch("knn_l2_tc rerank");
}

}  // extern "C"
