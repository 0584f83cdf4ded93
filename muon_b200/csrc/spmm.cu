// K2/K3 -- CSR x dense SpMM  C[n x P] (+)= A[n x d] * B[d x P]  for sm_90a, P in {32,64,128}.
//
// Replaces the per-Lanczos-step csr_matvec/csc_matvec pair that ARPACK drives inside
// scipy.sparse.linalg.svds (scipy _svds.py:428-460, called at muon/_atac/tools.py:53) by a
// blocked operator application on P vectors at once, and mofapy2's dense Y^T Z / Y W
// contractions (muon/_core/tools.py:583-585).  A^T * Y uses the same kernel on the CSR of
// A^T (transpose.cu).
//
// "Row-warp" kernel: a warp owns a row.  The dense operand B is fp32 or IEEE half (T).  Every lane
// gathers 16 B of a row of B, VEC = 16 / sizeof(T) values, so P/VEC lanes cover one row and a warp
// consumes G = 32 / (P/VEC) non-zeros per gather instruction.  Column indices and values are streamed
// in coalesced 128 B segments (32 per warp load, L1::no_allocate) and broadcast by shuffle; up to 16
// independent gathers are in flight per lane.  fp32 FMA accumulation in registers, 16 B stores per
// lane at the end of the row.
//
// Traffic model (DESIGN.md): HBM streams 8 B/nnz (+ dense operands once); every non-zero
// additionally pulls P * sizeof(T) bytes of B through L2->L1, which is the practical limiter at P>=32.
//
// "Tiled" kernel, for rows known to be sorted by column (CSR arrays or pairs) and the fp32 operand: a CTA owns a band
// of kTiledRows consecutive rows and sweeps B in column tiles (TC consecutive rows of B, one contiguous slab), each
// staged once into shared memory by a 1-D bulk copy (TMA) and shared by every row of the band.  Each operand row then
// leaves L2 once per band instead of once per non-zero, and the gathers are served from shared memory.  A warp keeps
// W rows' accumulators in registers and a 32-entry window of each row's (index, value) stream; the ballot of
// "column < tile end" over the window gives the row's segment in the tile.  The band's rows go to the warps by length
// (longest first, dealt snake-wise), so that no warp holds up the release of every tile.  Entry q of a row goes to
// lane group q mod G in ascending q, as in the row-warp kernel, and the butterfly and store are the same: a row's
// sum does not depend on the warp that owns it, and both kernels return the same bits.
//
// Half operand: every non-zero gathers half the bytes of the fp32 kernel.  Products and sums are fp32
// (half -> float conversion is exact), only the operand is rounded (2^-11 relative).  Used by the early
// block-Lanczos steps of the LSI driver (_lsi.py), whose accuracy need not exceed 1e-3; the final steps
// use the fp32 operand.  out_scale undoes the power-of-two scaling the caller applied before rounding
// (mub_f32_to_f16_scaled).
#include <cuda_fp16.h>

#include <climits>
#include <type_traits>

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

// acc[i] += v * (i-th value of the 16 B gather q)
template <typename T>
__device__ __forceinline__ void fma_gather(float* acc, float v, const uint4& q) {
    const unsigned w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        if constexpr (std::is_same_v<T, float>) {
            acc[i] = fmaf(v, __uint_as_float(w[i]), acc[i]);
        } else {
            const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
            acc[2 * i] = fmaf(v, f.x, acc[2 * i]);
            acc[2 * i + 1] = fmaf(v, f.y, acc[2 * i + 1]);
        }
    }
}

// combine the G lane groups of a row's partial sums (fixed butterfly order: deterministic) and store the row
template <int P, typename T>
__device__ __forceinline__ void store_row(float* acc, float* __restrict__ C_row, int accumulate, float out_scale,
                                          int lane) {
    constexpr int VEC = 16 / sizeof(T);
    constexpr int LPN = P / VEC;
    const int sub = lane % LPN, grp = lane / LPN;
#pragma unroll
    for (int off = LPN; off < 32; off <<= 1) {
#pragma unroll
        for (int i = 0; i < VEC; ++i) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], off);
    }
    if (grp == 0) {
        float4* dst = reinterpret_cast<float4*>(C_row + sub * VEC);
#pragma unroll
        for (int j = 0; j < VEC / 4; ++j) {
            float4 r = make_float4(acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3]);
            if constexpr (std::is_same_v<T, __half>) {
                // __fmul_rn is never contracted with the add below: the scaled product is rounded on its own, as it
                // is without accumulate
                r.x = __fmul_rn(r.x, out_scale); r.y = __fmul_rn(r.y, out_scale);
                r.z = __fmul_rn(r.z, out_scale); r.w = __fmul_rn(r.w, out_scale);
            }
            if (accumulate) {
                const float4 o = dst[j];
                r.x += o.x; r.y += o.y; r.z += o.z; r.w += o.w;
            }
            dst[j] = r;
        }
    }
}

template <int P, bool PAIRS, typename T>
__device__ __forceinline__ void spmm_row(const int32_t* __restrict__ indices, const float* __restrict__ data,
                                         int64_t start, int64_t end, const T* __restrict__ B,
                                         float* __restrict__ C_row, int accumulate, float out_scale, int lane) {
    constexpr int VEC = 16 / sizeof(T);            // values per 16 B gather
    constexpr int LPN = P / VEC;                   // lanes per non-zero
    constexpr int G = 32 / LPN;                    // non-zeros per warp-wide gather
    constexpr int STEPS = 32 / G;                  // gathers per 32-nnz segment
    constexpr int BATCH = STEPS < 16 ? STEPS : 16; // gathers in flight per lane
    const int sub = lane % LPN, grp = lane / LPN;
    const T* Bl = B + sub * VEC;
    float acc[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) acc[i] = 0.f;
    int64_t base = start;
    // full 32-nnz segments.  The (index, value) stream comes from HBM (~600 ns), the gathers from L2 (~130 ns):
    // the NEXT segment's entries are requested before the gathers of the current one, so a warp never waits for
    // both latencies in sequence
    int c_next = 0;
    float v_next = 0.f;
    bool more = base + 32 <= end;
    if (more) load_entry<PAIRS>(indices, data, base + lane, c_next, v_next);
    for (; more; base += 32) {
        const int c = c_next;
        const float v = v_next;
        more = base + 64 <= end;
        if (more) load_entry<PAIRS>(indices, data, base + 32 + lane, c_next, v_next);
#pragma unroll
        for (int t0 = 0; t0 < STEPS; t0 += BATCH) {
            uint4 b[BATCH];
            float vv[BATCH];
#pragma unroll
            for (int t = 0; t < BATCH; ++t) {
                const int cc = __shfl_sync(0xffffffffu, c, (t0 + t) * G + grp);
                vv[t] = __shfl_sync(0xffffffffu, v, (t0 + t) * G + grp);
                b[t] = ld_gather_u4(Bl + (size_t)cc * P);
            }
#pragma unroll
            for (int t = 0; t < BATCH; ++t) fma_gather<T>(acc, vv[t], b[t]);
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
            const int src = t * G + grp;  // < 32: G divides 32 and cnt < 32
            const int cc = __shfl_sync(0xffffffffu, c, src);
            const float vt = __shfl_sync(0xffffffffu, v, src);
            if (src < cnt) fma_gather<T>(acc, vt, ld_gather_u4(Bl + (size_t)cc * P));
        }
    }
    store_row<P, T>(acc, C_row, accumulate, out_scale, lane);
}

template <int P, bool PAIRS, typename T>
__global__ void __launch_bounds__(kSpmmThreads)
spmm_csr_rowwarp_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                        const float* __restrict__ data, int64_t n_rows, const T* __restrict__ B,
                        float* __restrict__ C, int accumulate, float out_scale, unsigned long long* row_counter) {
    const int lane = threadIdx.x & 31;
    if (row_counter == nullptr) {
        const int64_t warp = (int64_t)blockIdx.x * kSpmmWarps + (threadIdx.x >> 5);
        const int64_t n_warps = (int64_t)gridDim.x * kSpmmWarps;
        for (int64_t row = warp; row < n_rows; row += n_warps) {
            const int64_t s = __ldg(indptr + row), e = __ldg(indptr + row + 1);
            spmm_row<P, PAIRS, T>(indices, data, s, e, B, C + (size_t)row * P, accumulate, out_scale, lane);
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
            spmm_row<P, PAIRS, T>(indices, data, s, e, B, C + (size_t)row * P, accumulate, out_scale, lane);
        }
    }
}

template <int P, bool PAIRS, typename T>
static int launch_spmm(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_rows,
                       const T* B, float* C, int accumulate, float out_scale, unsigned long long* row_counter,
                       cudaStream_t stream, const char* name) {
    int64_t want = (n_rows + kSpmmWarps - 1) / kSpmmWarps;
    int64_t cap = (int64_t)sm_count() * 8;  // 2048 threads / SM
    int grid = (int)(want < cap ? want : cap);
    if (grid < 1) grid = 1;
    spmm_csr_rowwarp_kernel<P, PAIRS, T><<<grid, kSpmmThreads, 0, stream>>>(indptr, indices, data, n_rows, B, C,
                                                                          accumulate, out_scale, row_counter);
    return check_launch(name);
}

// ---- tiled kernel ------------------------------------------------------------------------------------------------
// Sorted rows and the fp32 operand only (see spmm_entry).  NW warps x W rows = a band of 128 rows per CTA, one CTA per
// SM (NW * 32 threads; a row's partial sums are 4 registers per lane).  Two stages of kTiledStageBytes: TC =
// kTiledStageBytes / (4 P) rows of B per tile.  The kernel's time is a fixed part plus a cost per (row, tile) segment,
// so the tiles are as tall as two stages allow next to the L1 that caches the entry windows.
constexpr int kTiledWarps = 16;
constexpr int kTiledRowsPerWarp = 8;
constexpr int kTiledRows = 128;
constexpr int kTiledStages = 2;
constexpr int kTiledStageBytes = 96 << 10;  // TC = 384 rows of B at P = 64: ~12 entries per segment at 3 % density
constexpr int kTiledSmemBytes = kTiledStages * kTiledStageBytes;
static_assert(kTiledWarps * kTiledRowsPerWarp == kTiledRows, "a band is NW x W rows");

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_addr(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, unsigned parity) {
    asm volatile(
        "{\n\t.reg .pred done;\n"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 done, [%0], %1;\n\t"
        "@!done bra WAIT_%=;\n}" ::"r"(smem_addr(bar)), "r"(parity) : "memory");
}
// bytes of B[src, src + bytes) -> shared dst; completion is counted on bar
__device__ __forceinline__ void tma_load_1d(void* dst, const void* src, unsigned bytes, uint64_t* bar) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_addr(dst)), "l"(src), "r"(bytes), "r"(smem_addr(bar)) : "memory");
}

// lane j <- entry pos + j of the row [start, start + len), column INT_MAX past the row's end.  Cached loads: the part
// of the window a tile does not consume is read again at the next tile
template <bool PAIRS>
__device__ __forceinline__ void load_window(const int32_t* __restrict__ indices, const float* __restrict__ data,
                                            int64_t start, int pos, int len, int lane, int& c, float& v) {
    c = INT_MAX;
    v = 0.f;
    if (pos + lane < len) {
        if constexpr (PAIRS) {
            const int2 e = __ldg(reinterpret_cast<const int2*>(indices) + start + pos + lane);
            c = e.x;
            v = __int_as_float(e.y);
        } else {
            c = __ldg(indices + start + pos + lane);
            v = __ldg(data + start + pos + lane);
        }
    }
}

// The band's rows dealt to warps by length: rank the R rows from the longest down (ties: lower row first; rows past
// n_rows rank last) and deal the ranks snake-wise, rank p to warp p mod NW in even rounds and NW - 1 - p mod NW in odd
// ones, round p / NW being the slot.  A tile is released only when every warp is done with it, so it runs at the pace
// of the warp with the most entries in it; dealt this way each warp's rows sum to about the band's mean.  Every warp
// ranks all R rows itself (shuffles only, no CTA barrier).  Returns, in lane w < W, the row of slot w of this warp.
template <int NW, int W>
__device__ __forceinline__ int64_t band_row_of_slot(const int64_t* __restrict__ indptr, int64_t n_rows, int64_t band0,
                                                    int warp, int lane) {
    constexpr int K = NW * W / 32;  // rows per lane: lane l holds band rows l, l + 32, ...
    int len[K], rank[K];
#pragma unroll
    for (int k = 0; k < K; ++k) {
        const int64_t r = band0 + lane + 32 * k;
        len[k] = r < n_rows ? (int)(__ldg(indptr + r + 1) - __ldg(indptr + r)) : -1;
        rank[k] = 0;
    }
#pragma unroll
    for (int kk = 0; kk < K; ++kk) {
        for (int src = 0; src < 32; ++src) {
            const int lj = __shfl_sync(0xffffffffu, len[kk], src);
            const int j = src + 32 * kk;
#pragma unroll
            for (int k = 0; k < K; ++k) rank[k] += (lj > len[k]) | ((lj == len[k]) & (j < lane + 32 * k));
        }
    }
    int64_t row = 0;
#pragma unroll
    for (int w = 0; w < W; ++w) {
        const int p = w * NW + ((w & 1) ? NW - 1 - warp : warp);
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const unsigned m = __ballot_sync(0xffffffffu, rank[k] == p);
            if (m != 0u && lane == w) row = band0 + 32 * k + __ffs(m) - 1;
        }
    }
    return row;
}

// window lanes [0, cnt) hold row entries pos .. pos + cnt - 1, all in the staged tile (first row of B: lo):
// entry q goes to lane group q mod G, in ascending q
template <int P, typename T>
__device__ __forceinline__ void gather_segment(float* acc, const T* __restrict__ tile, int lo, int c, float v, int pos,
                                               int cnt, int lane) {
    constexpr int VEC = 16 / sizeof(T);
    constexpr int LPN = P / VEC;
    constexpr int G = 32 / LPN;
    constexpr int BATCH = 4;  // gathers in flight per lane (a segment is ~0.03 * TC / G ~ 4 gathers)
    const int sub = lane % LPN;
    const int first = ((lane / LPN) - pos) & (G - 1);  // this group's first window lane
    const T* tl = tile + sub * VEC;
    for (int k0 = 0; k0 < cnt; k0 += BATCH * G) {  // warp-uniform trip count: the loop holds shuffles
        uint4 b[BATCH];
        float vv[BATCH];
#pragma unroll
        for (int t = 0; t < BATCH; ++t) {
            const int j = k0 + t * G + first;
            const int cc = __shfl_sync(0xffffffffu, c, j & 31);
            vv[t] = __shfl_sync(0xffffffffu, v, j & 31);
            if (j < cnt) b[t] = *reinterpret_cast<const uint4*>(tl + (cc - lo) * P);
        }
#pragma unroll
        for (int t = 0; t < BATCH; ++t)
            if (k0 + t * G + first < cnt) fma_gather<T>(acc, vv[t], b[t]);
    }
}

// PAIRS: interleaved (column, value) pairs, as in the row-warp kernel (the transposed panels)
template <int P, bool PAIRS, int NW, int W>
__global__ void __launch_bounds__(NW * kWarp, 1)
spmm_csr_tiled_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                      const float* __restrict__ data, int64_t n_rows, int n_cols, const float* __restrict__ B,
                      float* __restrict__ C, int accumulate) {
    using T = float;
    constexpr int VEC = 16 / sizeof(T);
    constexpr int TC = kTiledStageBytes / (P * (int)sizeof(T));
    constexpr int R = NW * W;
    constexpr int S = kTiledStages;
    static_assert(R % 32 == 0 && W <= 32, "band rows are ranked 32 per lane slot");
    extern __shared__ __align__(128) unsigned char stages[];
    __shared__ __align__(8) uint64_t full[S], empty[S];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int n_tiles = (n_cols + TC - 1) / TC;
    const int64_t n_bands = (n_rows + R - 1) / R;
    // bands blockIdx.x, blockIdx.x + gridDim.x, ...: one (band, tile) item after the other, the stages cycling
    // through all of them, so the next band's first tiles load under the current band's last ones
    const int64_t items = (n_bands - 1 - blockIdx.x) / gridDim.x * n_tiles + n_tiles;
    auto issue = [&](int64_t i) {
        const int lo = (int)(i % n_tiles) * TC;
        const unsigned bytes = (unsigned)(min(TC, n_cols - lo) * P * (int)sizeof(T));
        tma_load_1d(stages + (i % S) * kTiledStageBytes, B + (size_t)lo * P, bytes, &full[i % S]);
    };
    if (threadIdx.x == 0) {
        for (int s = 0; s < S; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], NW);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        for (int64_t i = 0; i < S && i < items; ++i) issue(i);
    }
    __syncthreads();

    float acc[W][VEC];
    int c[W];        // window of row w: lane j holds entry rpos(w) + j
    float v[W];
    int64_t row = 0;     // lane w < W: the row of slot w, its first entry, length and consumed entries
    int64_t rstart = 0;
    int rlen = 0, rpos = 0;
    for (int64_t i = 0; i < items; ++i) {
        const int tile = (int)(i % n_tiles);
        if (tile == 0) {
            const int64_t band0 = (blockIdx.x + i / n_tiles * gridDim.x) * (int64_t)R;
            row = band_row_of_slot<NW, W>(indptr, n_rows, band0, warp, lane);
            rstart = 0;
            rlen = rpos = 0;
            if (lane < W && row < n_rows) {
                rstart = __ldg(indptr + row);
                rlen = (int)(__ldg(indptr + row + 1) - rstart);
            }
#pragma unroll
            for (int w = 0; w < W; ++w) {
#pragma unroll
                for (int e = 0; e < VEC; ++e) acc[w][e] = 0.f;
                load_window<PAIRS>(indices, data, __shfl_sync(0xffffffffu, rstart, w), 0,
                                   __shfl_sync(0xffffffffu, rlen, w), lane, c[w], v[w]);
            }
        }
        const int s = (int)(i % S);
        mbar_wait(&full[s], (unsigned)(i / S) & 1u);
        const T* tl = reinterpret_cast<const T*>(stages + s * kTiledStageBytes);
        const int lo = tile * TC, hi = min(lo + TC, n_cols);
#pragma unroll
        for (int w = 0; w < W; ++w) {
            // sorted rows: the window's entries below hi are its first cnt lanes
            int cnt = __popc(__ballot_sync(0xffffffffu, c[w] < hi));
            if (cnt == 0) continue;
            int pos = __shfl_sync(0xffffffffu, rpos, w);
            const int64_t st = __shfl_sync(0xffffffffu, rstart, w);
            const int len = __shfl_sync(0xffffffffu, rlen, w);
            for (;;) {
                gather_segment<P, T>(acc[w], tl, lo, c[w], v[w], pos, cnt, lane);
                pos += cnt;
                load_window<PAIRS>(indices, data, st, pos, len, lane, c[w], v[w]);
                if (cnt < 32) break;  // the reload is only needed at the next tile
                cnt = __popc(__ballot_sync(0xffffffffu, c[w] < hi));
                if (cnt == 0) break;
            }
            if (lane == w) rpos = pos;
        }
        // release the stage; warp 0 refills it with item i + S once all warps have
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
        if (threadIdx.x == 0 && i + S < items) {
            mbar_wait(&empty[s], (unsigned)(i / S) & 1u);
            issue(i + S);
        }
        __syncwarp();
        if (tile == n_tiles - 1) {
#pragma unroll
            for (int w = 0; w < W; ++w) {
                const int64_t r = __shfl_sync(0xffffffffu, row, w);
                if (r < n_rows) store_row<P, T>(acc[w], C + (size_t)r * P, accumulate, 1.f, lane);
            }
        }
    }
}

template <int P, bool PAIRS>
static int launch_spmm_tiled(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_rows,
                             int n_cols, const float* B, float* C, int accumulate, cudaStream_t stream,
                             const char* name) {
    auto kernel = spmm_csr_tiled_kernel<P, PAIRS, kTiledWarps, kTiledRowsPerWarp>;
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kTiledSmemBytes);
    MUB_REQUIRE(e == cudaSuccess, "%s: %s", name, cudaGetErrorString(e));
    const int64_t bands = (n_rows + kTiledRows - 1) / kTiledRows;
    // one CTA per SM, every CTA sweeping B at about the same pace: the tiles a CTA stages were just staged by the
    // others and are still in L2
    const int grid = (int)(bands < sm_count() ? bands : sm_count());
    kernel<<<grid, kTiledWarps * kWarp, kTiledSmemBytes, stream>>>(indptr, indices, data, n_rows, n_cols, B, C,
                                                                   accumulate);
    return check_launch(name);
}

// the four C entry points: shared validation, then one instantiation per ld and schedule
template <bool PAIRS, typename T>
static int spmm_entry(const char* name, const int64_t* indptr, const int32_t* indices, const float* data,
                      int64_t n_rows, int64_t n_cols, const void* B, int32_t ld, float* C, int32_t accumulate,
                      float out_scale, unsigned long long* row_counter, uint32_t flags, mub_stream_t stream) {
    MUB_REQUIRE(n_rows >= 0 && n_cols >= 0, "%s: negative shape", name);
    MUB_REQUIRE(ld == 32 || ld == 64 || ld == 128, "%s: ld must be 32, 64 or 128 (got %d)", name, ld);
    MUB_REQUIRE((flags & ~(uint32_t)MUB_SPMM_ROWS_SORTED) == 0, "%s: unknown flags 0x%x", name, flags);
    if (n_rows == 0) return 0;
    MUB_REQUIRE(indptr && B && C, "%s: null pointer", name);
    MUB_REQUIRE((((uintptr_t)B | (uintptr_t)C) & 15) == 0, "%s: B and C must be 16-byte aligned", name);
    MUB_REQUIRE(!PAIRS || ((uintptr_t)indices & 7) == 0, "%s: pairs must be 8-byte aligned", name);
    const T* Bt = (const T*)B;
    cudaStream_t s = (cudaStream_t)stream;
    // measured on the LSI products (profiles/README.md): with the fp32 operand the tiled kernel wins on A*V and on the
    // pairs-layout A^T panels.  With the half operand the row-warp kernel gathers half the bytes while the tiled
    // kernel's cost per (row, tile) segment stays.  A launch of fewer bands than SMs (the sampled row blocks of the
    // residual check) would leave most SMs idle in the tiled kernel; the row-warp kernel spreads it over all of them
    if constexpr (std::is_same_v<T, float>) {
        if ((flags & MUB_SPMM_ROWS_SORTED) && n_cols > 0 && (n_rows + kTiledRows - 1) / kTiledRows >= sm_count()) {
            MUB_REQUIRE(n_cols < INT_MAX, "%s: n_cols must be below 2^31", name);
            const int d = (int)n_cols;
            switch (ld) {
                case 32: return launch_spmm_tiled<32, PAIRS>(indptr, indices, data, n_rows, d, Bt, C, accumulate, s, name);
                case 64: return launch_spmm_tiled<64, PAIRS>(indptr, indices, data, n_rows, d, Bt, C, accumulate, s, name);
                default: return launch_spmm_tiled<128, PAIRS>(indptr, indices, data, n_rows, d, Bt, C, accumulate, s, name);
            }
        }
    }
    switch (ld) {
        case 32: return launch_spmm<32, PAIRS, T>(indptr, indices, data, n_rows, Bt, C, accumulate, out_scale, row_counter, s, name);
        case 64: return launch_spmm<64, PAIRS, T>(indptr, indices, data, n_rows, Bt, C, accumulate, out_scale, row_counter, s, name);
        default: return launch_spmm<128, PAIRS, T>(indptr, indices, data, n_rows, Bt, C, accumulate, out_scale, row_counter, s, name);
    }
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

}  // namespace mub

extern "C" int mub_spmm_csr_f32(const int64_t* indptr, const int32_t* indices, const float* data,
                                int64_t n_rows, int64_t n_cols, const float* B, int32_t ld, float* C,
                                int32_t accumulate, unsigned long long* row_counter, uint32_t flags,
                                mub_stream_t stream) {
    return mub::spmm_entry<false, float>("spmm_csr", indptr, indices, data, n_rows, n_cols, B, ld, C, accumulate, 1.f,
                                         row_counter, flags, stream);
}

extern "C" int mub_spmm_csrp_f32(const int64_t* indptr, const int32_t* pairs, int64_t n_rows, int64_t n_cols,
                                 const float* B, int32_t ld, float* C, int32_t accumulate,
                                 unsigned long long* row_counter, uint32_t flags, mub_stream_t stream) {
    return mub::spmm_entry<true, float>("spmm_csrp", indptr, pairs, nullptr, n_rows, n_cols, B, ld, C, accumulate, 1.f,
                                        row_counter, flags, stream);
}

extern "C" int mub_spmm_csr_h16(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_rows,
                                int64_t n_cols, const void* B_half, int32_t ld, float* C, int32_t accumulate,
                                float out_scale, unsigned long long* row_counter, uint32_t flags,
                                mub_stream_t stream) {
    return mub::spmm_entry<false, __half>("spmm_csr_h16", indptr, indices, data, n_rows, n_cols, B_half, ld, C,
                                          accumulate, out_scale, row_counter, flags, stream);
}

extern "C" int mub_spmm_csrp_h16(const int64_t* indptr, const int32_t* pairs, int64_t n_rows, int64_t n_cols,
                                 const void* B_half, int32_t ld, float* C, int32_t accumulate, float out_scale,
                                 unsigned long long* row_counter, uint32_t flags, mub_stream_t stream) {
    return mub::spmm_entry<true, __half>("spmm_csrp_h16", indptr, pairs, nullptr, n_rows, n_cols, B_half, ld, C,
                                         accumulate, out_scale, row_counter, flags, stream);
}

extern "C" int mub_f32_to_f16_scaled(const float* src, int64_t n, float scale, void* dst, mub_stream_t stream) {
    MUB_REQUIRE(n >= 0 && (n % 4) == 0, "f32_to_f16_scaled: n must be a non-negative multiple of 4");
    if (n == 0) return 0;
    MUB_REQUIRE(src && dst && (((uintptr_t)src & 15) == 0) && (((uintptr_t)dst & 7) == 0), "f32_to_f16_scaled: misaligned operand");
    int64_t want = (n / 4 + 255) / 256, cap = (int64_t)mub::sm_count() * 8;
    int grid = (int)(want < cap ? want : cap);
    mub::f32_to_f16_scaled_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const float4*)src, n / 4, scale, (uint2*)dst);
    return mub::check_launch("f32_to_f16_scaled");
}
