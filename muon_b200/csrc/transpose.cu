// CSR -> CSR-of-transpose (one-time per matrix) so that A^T * Y is a row-gather SpMM too.
// scipy reaches the same effect through csc_matvec on the CSR arrays (_svds.py:447 via
// muon/_atac/tools.py:53); on the GPU a scatter-add formulation would need ld atomics per
// non-zero, so the transposed copy is built once per LSI/MOFA call instead.
//
// count : histogram of column indices (int64 counters, one red per non-zero, L2-resident)
// fill  : warp per source row; each non-zero claims a slot in its column with an atomic
//         cursor (seeded from the scanned histogram) and writes (row, value) there.
#include "common.cuh"

namespace mub {

__global__ void __launch_bounds__(256)
transpose_count_kernel(const int32_t* __restrict__ indices, int64_t nnz, int head,
                       unsigned long long* t_count) {
    // `head` leading elements (<4) precede the first 16-byte boundary: scalar path
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < head) atomicAdd(t_count + 1 + ld_stream(indices + i), 1ull);
    indices += head;
    nnz -= head;
    const int64_t nvec = nnz >> 2;
    const int4* v = reinterpret_cast<const int4*>(indices);
    for (int64_t k = i; k < nvec; k += stride) {
        const int4 c = ld_stream4(v + k);
        atomicAdd(t_count + 1 + c.x, 1ull);
        atomicAdd(t_count + 1 + c.y, 1ull);
        atomicAdd(t_count + 1 + c.z, 1ull);
        atomicAdd(t_count + 1 + c.w, 1ull);
    }
    for (int64_t k = (nvec << 2) + i; k < nnz; k += stride) atomicAdd(t_count + 1 + ld_stream(indices + k), 1ull);
}

__global__ void copy_i64_kernel(const int64_t* __restrict__ src, int64_t* __restrict__ dst, int64_t n) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = src[i];
}

__global__ void __launch_bounds__(256)
transpose_fill_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                      const float* __restrict__ data, int64_t n_rows, int64_t row_offset,
                      unsigned long long* cursor, int32_t* __restrict__ t_indices, float* __restrict__ t_data) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int64_t n_warps = (int64_t)gridDim.x * 8;
    for (int64_t row = warp; row < n_rows; row += n_warps) {
        const int64_t s = __ldg(indptr + row), e = __ldg(indptr + row + 1);
        const int32_t r = (int32_t)(row + row_offset);
        int64_t k = s + lane;
        // 4 independent slot claims in flight per lane (the atomic's return latency dominates)
        for (; k + 96 < e; k += 128) {
            const int c0 = ld_stream(indices + k), c1 = ld_stream(indices + k + 32);
            const int c2 = ld_stream(indices + k + 64), c3 = ld_stream(indices + k + 96);
            const float v0 = ld_stream(data + k), v1 = ld_stream(data + k + 32);
            const float v2 = ld_stream(data + k + 64), v3 = ld_stream(data + k + 96);
            const unsigned long long s0 = atomicAdd(cursor + c0, 1ull), s1 = atomicAdd(cursor + c1, 1ull);
            const unsigned long long s2 = atomicAdd(cursor + c2, 1ull), s3 = atomicAdd(cursor + c3, 1ull);
            t_indices[s0] = r; t_data[s0] = v0;
            t_indices[s1] = r; t_data[s1] = v1;
            t_indices[s2] = r; t_data[s2] = v2;
            t_indices[s3] = r; t_data[s3] = v3;
        }
        for (; k < e; k += 32) {
            const int c = ld_stream(indices + k);
            const float v = ld_stream(data + k);
            const unsigned long long slot = atomicAdd(cursor + c, 1ull);
            t_indices[slot] = r;
            t_data[slot] = v;
        }
    }
}

// Same scatter, but (row, value) is written as ONE 8-byte pair: one scattered store per non-zero instead of
// two (the fill is bound by the rate of scattered L2 operations, not by bytes).
__global__ void __launch_bounds__(256)
transpose_fill_pairs_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                            const float* __restrict__ data, int64_t n_rows, int64_t row_offset,
                            unsigned long long* cursor, int2* __restrict__ t_pairs) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int64_t n_warps = (int64_t)gridDim.x * 8;
    for (int64_t row = warp; row < n_rows; row += n_warps) {
        const int64_t s = __ldg(indptr + row), e = __ldg(indptr + row + 1);
        const int32_t r = (int32_t)(row + row_offset);
        int64_t k = s + lane;
        for (; k + 96 < e; k += 128) {
            const int c0 = ld_stream(indices + k), c1 = ld_stream(indices + k + 32);
            const int c2 = ld_stream(indices + k + 64), c3 = ld_stream(indices + k + 96);
            const float v0 = ld_stream(data + k), v1 = ld_stream(data + k + 32);
            const float v2 = ld_stream(data + k + 64), v3 = ld_stream(data + k + 96);
            const unsigned long long s0 = atomicAdd(cursor + c0, 1ull), s1 = atomicAdd(cursor + c1, 1ull);
            const unsigned long long s2 = atomicAdd(cursor + c2, 1ull), s3 = atomicAdd(cursor + c3, 1ull);
            t_pairs[s0] = make_int2(r, __float_as_int(v0));
            t_pairs[s1] = make_int2(r, __float_as_int(v1));
            t_pairs[s2] = make_int2(r, __float_as_int(v2));
            t_pairs[s3] = make_int2(r, __float_as_int(v3));
        }
        for (; k < e; k += 32) {
            const int c = ld_stream(indices + k);
            const float v = ld_stream(data + k);
            t_pairs[atomicAdd(cursor + c, 1ull)] = make_int2(r, __float_as_int(v));
        }
    }
}

// ---- tiled fill: no global atomics, deterministic ------------------------------------------------------------
// The atomic-cursor fill above spends one global ATOM (with return) plus one scattered 8-byte store per non-zero,
// and the order in which slots are claimed -- hence the order of the entries inside a transposed row, hence the fp32
// summation order of every A^T Y product -- changes from run to run.  When the TF-IDF reduce pass has left the
// entry count of every (512-row block, column) behind (tfidf.cu, rb_count), the write offset of block b in column c
// is  t_indptr[c] + sum of the counts of the panel's earlier blocks  -- a column-wise scan.  Inside its block a CTA
// sweeps the columns tile by tile; warp w owns the 32 consecutive rows [32w, 32w + 32) and walks them in order.
// Per tile it first counts its entries per column (the columns of one row are distinct, so the lanes never collide),
// the counts are scanned over the warps in warp order, and a second walk writes every entry at the next slot of its
// (warp, column) cursor.  Every transposed row therefore lists its cells in ascending order, on every run.
constexpr int kFillTileCols = 2048;    // 16 warps x 2048 columns x 4 B = 128 KB of per-warp cursors
constexpr int kFillRows = 512;         // must equal the reduce kernel's block height (mub_tfidf_tile_rows)
constexpr int kFillThreads = 512;
constexpr int kFillWarps = kFillThreads / 32;
constexpr int kFillRowsPerWarp = kFillRows / kFillWarps;

// base[b][c] = t_indptr[c] + sum_{b' < b} count[b'][c] for the blocks of one panel (one thread per column)
__global__ void __launch_bounds__(256)
transpose_scan_blocks_kernel(const uint16_t* __restrict__ rb_count, int32_t n_cols, int64_t n_blocks,
                             const int64_t* __restrict__ t_indptr, uint32_t* __restrict__ base, int* __restrict__ status) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n_cols) return;
    unsigned long long run = (unsigned long long)t_indptr[c];
    for (int64_t b = 0; b < n_blocks; ++b) {
        base[(size_t)b * n_cols + c] = (uint32_t)run;
        run += rb_count[(size_t)b * n_cols + c];
    }
    if (run != (unsigned long long)t_indptr[c + 1] || run > 0xffffffffull) atomicOr(status, 1);   // counts and indptr disagree
}

__global__ void __launch_bounds__(kFillThreads, 1)
transpose_fill_tiled_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                            const float* __restrict__ data, int64_t n_rows, int32_t n_cols,
                            const uint32_t* __restrict__ base, int2* __restrict__ t_pairs) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint32_t* wcur = reinterpret_cast<uint32_t*>(smem_raw);                        // [kFillWarps][kFillTileCols]
    int* cur = reinterpret_cast<int*>(wcur + kFillWarps * kFillTileCols);           // [kFillRows] entries done per row
    int* ntile = cur + kFillRows;                                                   // [kFillRows] entries in this tile
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t r0 = (int64_t)blockIdx.x * kFillRows;
    const int rows_here = (int)((n_rows - r0) < kFillRows ? (n_rows - r0) : kFillRows);
    const int my_r0 = warp * kFillRowsPerWarp;
    const int my_r1 = (my_r0 + kFillRowsPerWarp < rows_here) ? my_r0 + kFillRowsPerWarp : rows_here;
    uint32_t* my_cur = wcur + warp * kFillTileCols;
    for (int r = threadIdx.x; r < kFillRows; r += kFillThreads) cur[r] = 0;
    const uint32_t* my_base = base + (size_t)blockIdx.x * n_cols;
    const int n_tiles = (n_cols + kFillTileCols - 1) / kFillTileCols;
    for (int t = 0; t < n_tiles; ++t) {
        const int c_lo = t * kFillTileCols;
        const int c_hi = (c_lo + kFillTileCols < n_cols) ? c_lo + kFillTileCols : n_cols;
        for (int j = threadIdx.x; j < kFillWarps * kFillTileCols; j += kFillThreads) wcur[j] = 0;
        __syncthreads();
        // walk 1: entries per (warp, column) of this tile, and per row the number of its entries inside the tile
        for (int r = my_r0; r < my_r1; ++r) {
            const int64_t e = __ldg(indptr + r0 + r + 1);
            const int64_t k0 = __ldg(indptr + r0 + r) + cur[r];
            int64_t k = k0;
            for (;;) {
                const int c = k + lane < e ? ld_stream(indices + k + lane) : 0x7fffffff;
                const bool in = c < c_hi;                  // sorted row: the entries of this tile come first
                const int n_in = __popc(__ballot_sync(0xffffffffu, in));
                if (in && c >= c_lo) my_cur[c - c_lo] += 1;
                k += n_in;
                if (n_in < 32) break;
            }
            if (lane == 0) ntile[r] = (int)(k - k0);
        }
        __syncthreads();
        // exclusive scan over the warps, in warp (= row) order, from the block's write offset of each column
        for (int j = threadIdx.x; j < c_hi - c_lo; j += kFillThreads) {
            uint32_t run = my_base[c_lo + j];
#pragma unroll
            for (int w = 0; w < kFillWarps; ++w) {
                const uint32_t cnt = wcur[w * kFillTileCols + j];
                wcur[w * kFillTileCols + j] = run;
                run += cnt;
            }
        }
        __syncthreads();
        // walk 2: rows in order, each entry at the next slot of its (warp, column) cursor
        for (int r = my_r0; r < my_r1; ++r) {
            const int64_t k0 = __ldg(indptr + r0 + r) + cur[r];
            const int n = ntile[r];
            for (int i = lane; i < n; i += 32) {
                const int c = ld_stream(indices + k0 + i);
                const float v = ld_stream(data + k0 + i);
                if (c >= c_lo) {
                    const uint32_t slot = my_cur[c - c_lo]++;
                    t_pairs[slot] = make_int2((int)(r0 + r), __float_as_int(v));
                }
            }
            __syncwarp();
            if (lane == 0) cur[r] += n;
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256)
row_stats_pairs_kernel(const int64_t* __restrict__ indptr, const int2* __restrict__ pairs, int64_t n_rows,
                       double* __restrict__ sum, double* __restrict__ sumsq) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int64_t n_warps = (int64_t)gridDim.x * 8;
    for (int64_t row = warp; row < n_rows; row += n_warps) {
        const int64_t s = __ldg(indptr + row), e = __ldg(indptr + row + 1);
        double a = 0.0, b = 0.0;
        for (int64_t k = s + lane; k < e; k += 32) {
            const double v = (double)__int_as_float(ld_stream2(pairs + k).y);
            a += v;
            b += v * v;
        }
        a = warp_sum(a);
        b = warp_sum(b);
        if (lane == 0) {
            sum[row] = a;
            sumsq[row] = b;
        }
    }
}

// per-row sum and sum of squares (fp64 accumulation); applied to the CSR of A^T this yields
// the per-feature moments MOFA's centring needs (intercepts, muon/_core/tools.py:283-286)
__global__ void __launch_bounds__(256)
row_stats_kernel(const int64_t* __restrict__ indptr, const float* __restrict__ data, int64_t n_rows,
                 double* __restrict__ sum, double* __restrict__ sumsq) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int64_t n_warps = (int64_t)gridDim.x * 8;
    for (int64_t row = warp; row < n_rows; row += n_warps) {
        const int64_t s = __ldg(indptr + row), e = __ldg(indptr + row + 1);
        double a = 0.0, b = 0.0;
        for (int64_t k = s + lane; k < e; k += 32) {
            const double v = (double)ld_stream(data + k);
            a += v;
            b += v * v;
        }
        a = warp_sum(a);
        b = warp_sum(b);
        if (lane == 0) {
            sum[row] = a;
            sumsq[row] = b;
        }
    }
}

}  // namespace mub

extern "C" {

int mub_csr_transpose_fill_pairs(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_rows,
                                 int32_t n_cols, int64_t row_offset, const int64_t* t_indptr, int64_t* cursor,
                                 int32_t* t_pairs, mub_stream_t stream) {
    MUB_REQUIRE(n_rows >= 0 && n_cols >= 0, "transpose_fill_pairs: negative shape");
    if (n_rows == 0 || n_cols == 0) return 0;
    MUB_REQUIRE(indptr && t_indptr && cursor && t_pairs, "transpose_fill_pairs: null pointer");
    MUB_REQUIRE(((uintptr_t)t_pairs & 7) == 0, "transpose_fill_pairs: t_pairs must be 8-byte aligned");
    cudaStream_t s = (cudaStream_t)stream;
    mub::copy_i64_kernel<<<(n_cols + 255) / 256, 256, 0, s>>>(t_indptr, cursor, n_cols);
    int64_t want = (n_rows + 7) / 8;
    int64_t cap = (int64_t)mub::sm_count() * 8;
    int grid = (int)(want < cap ? want : cap);
    if (grid < 1) grid = 1;
    mub::transpose_fill_pairs_kernel<<<grid, 256, 0, s>>>(indptr, indices, data, n_rows, row_offset,
                                                         (unsigned long long*)cursor, (int2*)t_pairs);
    return mub::check_launch("transpose_fill_pairs");
}

int mub_csrp_row_stats_f32(const int64_t* indptr, const int32_t* pairs, int64_t n_rows, double* sum, double* sumsq,
                           mub_stream_t stream) {
    MUB_REQUIRE(n_rows >= 0, "csrp_row_stats: negative n_rows");
    if (n_rows == 0) return 0;
    MUB_REQUIRE(indptr && sum && sumsq, "csrp_row_stats: null pointer");
    int64_t want = (n_rows + 7) / 8, cap = (int64_t)mub::sm_count() * 8;
    int grid = (int)(want < cap ? want : cap);
    mub::row_stats_pairs_kernel<<<grid < 1 ? 1 : grid, 256, 0, (cudaStream_t)stream>>>(indptr, (const int2*)pairs,
                                                                                     n_rows, sum, sumsq);
    return mub::check_launch("csrp_row_stats");
}

int mub_csr_row_stats_f32(const int64_t* indptr, const float* data, int64_t n_rows, double* sum, double* sumsq,
                          mub_stream_t stream) {
    MUB_REQUIRE(n_rows >= 0, "csr_row_stats: negative n_rows");
    if (n_rows == 0) return 0;
    MUB_REQUIRE(indptr && sum && sumsq, "csr_row_stats: null pointer");
    int64_t want = (n_rows + 7) / 8, cap = (int64_t)mub::sm_count() * 8;
    int grid = (int)(want < cap ? want : cap);
    mub::row_stats_kernel<<<grid < 1 ? 1 : grid, 256, 0, (cudaStream_t)stream>>>(indptr, data, n_rows, sum, sumsq);
    return mub::check_launch("csr_row_stats");
}

int mub_csr_transpose_count(const int32_t* indices, int64_t nnz, int32_t n_cols, int64_t* t_count,
                            mub_stream_t stream) {
    MUB_REQUIRE(nnz >= 0 && n_cols >= 0, "transpose_count: negative size");
    if (nnz == 0) return 0;
    MUB_REQUIRE(indices && t_count, "transpose_count: null pointer");
    MUB_REQUIRE(((uintptr_t)indices & 3) == 0, "transpose_count: indices must be 4-byte aligned");
    int head = (int)(((16 - ((uintptr_t)indices & 15)) & 15) >> 2);
    if (head > nnz) head = (int)nnz;
    int64_t want = (nnz / 4 + 255) / 256;
    int64_t cap = (int64_t)mub::sm_count() * 8;
    int grid = (int)(want < cap ? want : cap);
    if (grid < 1) grid = 1;
    mub::transpose_count_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(indices, nnz, head,
                                                                      (unsigned long long*)t_count);
    return mub::check_launch("transpose_count");
}

int mub_csr_transpose_fill(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_rows,
                           int32_t n_cols, int64_t row_offset, const int64_t* t_indptr, int64_t* cursor,
                           int32_t* t_indices, float* t_data, mub_stream_t stream) {
    MUB_REQUIRE(n_rows >= 0 && n_cols >= 0, "transpose_fill: negative shape");
    if (n_rows == 0 || n_cols == 0) return 0;
    MUB_REQUIRE(indptr && t_indptr && cursor && t_indices && t_data, "transpose_fill: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    mub::copy_i64_kernel<<<(n_cols + 255) / 256, 256, 0, s>>>(t_indptr, cursor, n_cols);
    int64_t want = (n_rows + 7) / 8;
    int64_t cap = (int64_t)mub::sm_count() * 8;
    int grid = (int)(want < cap ? want : cap);
    if (grid < 1) grid = 1;
    mub::transpose_fill_kernel<<<grid, 256, 0, s>>>(indptr, indices, data, n_rows, row_offset,
                                                   (unsigned long long*)cursor, t_indices, t_data);
    return mub::check_launch("transpose_fill");
}

}  // extern "C"

// ---- tiled fill (needs the per-row-block counts of mub_tfidf_reduce_tiled_f32) ------------------------------------
extern "C" int mub_csr_transpose_fill_tiled(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_rows,
                                            int32_t n_cols, const uint16_t* rb_count, const int64_t* t_indptr, uint32_t* base,
                                            int32_t* t_pairs, int32_t* status, mub_stream_t stream) {
    MUB_REQUIRE(n_rows >= 0 && n_cols >= 0, "transpose_fill_tiled: negative shape");
    if (n_rows == 0 || n_cols == 0) return 0;
    MUB_REQUIRE(indptr && rb_count && t_indptr && base && t_pairs && status, "transpose_fill_tiled: null pointer");
    MUB_REQUIRE(((uintptr_t)t_pairs & 7) == 0, "transpose_fill_tiled: t_pairs must be 8-byte aligned");
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t n_blocks = (n_rows + mub::kFillRows - 1) / mub::kFillRows;
    MUB_REQUIRE(n_blocks < (1ll << 31), "transpose_fill_tiled: too many rows");
    mub::transpose_scan_blocks_kernel<<<(n_cols + 255) / 256, 256, 0, s>>>(rb_count, n_cols, n_blocks, t_indptr, base, status);
    const size_t smem = sizeof(uint32_t) * mub::kFillWarps * mub::kFillTileCols + 2 * sizeof(int) * mub::kFillRows;
    cudaError_t e = cudaFuncSetAttribute(mub::transpose_fill_tiled_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) {
        mub::set_error("transpose_fill_tiled: %zu B of shared memory: %s", smem, cudaGetErrorString(e));
        return -2;
    }
    mub::transpose_fill_tiled_kernel<<<(int)n_blocks, mub::kFillThreads, smem, s>>>(indptr, indices, data, n_rows, n_cols, base,
                                                                                  (int2*)t_pairs);
    return mub::check_launch("transpose_fill_tiled");
}
