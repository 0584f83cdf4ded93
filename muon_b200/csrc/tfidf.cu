// K1 -- fused CSR TF-IDF for sm_90a (reference arithmetic: muon/_atac/preproc.py:92-119).
//
// Two streaming passes over the CSR arrays, both HBM-bound:
//   reduce : reads indices+values (8 B/nnz fp32), warp-shuffle row sums, column sums by
//            red.global.add into an L2-resident D-vector (0.8 MB at D=200k)
//   apply  : reads indices+values, writes values (12 B/nnz fp32); idf[j] is gathered from
//            a D-vector that stays in L1/L2; 1/r_i computed once per row
// Algorithmic bytes: 20 B/nnz (fp32) + 8(n+1) + 8D  (SURVEY section 8d).
//
// One warp owns one row at a time (coalesced 128 B segments of indices and values, four
// independent segments in flight per lane); warps take rows round-robin so that
// consecutive warps stream consecutive memory.
#include <math.h>

#include "common.cuh"

namespace mub {

constexpr int kThreads = 256;
constexpr int kWarpsPerCta = kThreads / kWarp;

template <typename T, bool binarize>
__global__ void __launch_bounds__(kThreads)
tfidf_reduce_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                    const T* __restrict__ data, int64_t n_rows, T* __restrict__ row_sum,
                    T* __restrict__ col_sum, int* __restrict__ status) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (int64_t)blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5);
    const int64_t n_warps = (int64_t)gridDim.x * kWarpsPerCta;
    int bad = 0;  // bit0: indices not strictly increasing inside a row, bit1: explicit zero
    for (int64_t row = warp; row < n_rows; row += n_warps) {
        const int64_t start = __ldg(indptr + row), end = __ldg(indptr + row + 1);
        T acc = 0;
        int carry = -1;  // last column index of the previous 32-wide segment of this row
        // 4 independent coalesced segments in flight per lane; trip counts are warp-uniform
        // (the canonical-form check below shuffles across the whole warp)
        int64_t kb = start;
        for (; kb + 128 <= end; kb += 128) {
            const int64_t k = kb + lane;
            int c0 = ld_stream(indices + k), c1 = ld_stream(indices + k + 32);
            int c2 = ld_stream(indices + k + 64), c3 = ld_stream(indices + k + 96);
            T v0 = ld_stream(data + k), v1 = ld_stream(data + k + 32);
            T v2 = ld_stream(data + k + 64), v3 = ld_stream(data + k + 96);
            bad |= ((v0 == T(0)) | (v1 == T(0)) | (v2 == T(0)) | (v3 == T(0))) << 1;
            if (binarize) {
                v0 = v0 != T(0) ? T(1) : T(0); v1 = v1 != T(0) ? T(1) : T(0);
                v2 = v2 != T(0) ? T(1) : T(0); v3 = v3 != T(0) ? T(1) : T(0);
            }
            atomicAdd(col_sum + c0, v0);
            atomicAdd(col_sum + c1, v1);
            atomicAdd(col_sum + c2, v2);
            atomicAdd(col_sum + c3, v3);
            acc += (v0 + v1) + (v2 + v3);
            // canonical-form check: each index must exceed its predecessor in the row
            int p0 = __shfl_up_sync(0xffffffffu, c0, 1), p1 = __shfl_up_sync(0xffffffffu, c1, 1);
            int p2 = __shfl_up_sync(0xffffffffu, c2, 1), p3 = __shfl_up_sync(0xffffffffu, c3, 1);
            const int l0 = __shfl_sync(0xffffffffu, c0, 31), l1 = __shfl_sync(0xffffffffu, c1, 31);
            const int l2 = __shfl_sync(0xffffffffu, c2, 31), l3 = __shfl_sync(0xffffffffu, c3, 31);
            if (lane == 0) { p0 = carry; p1 = l0; p2 = l1; p3 = l2; }
            carry = l3;
            bad |= (c0 <= p0) | (c1 <= p1) | (c2 <= p2) | (c3 <= p3);
        }
        for (; kb < end; kb += 32) {
            const int64_t k = kb + lane;
            const bool ok = k < end;
            int c = ok ? ld_stream(indices + k) : 0x7fffffff;
            T v = ok ? ld_stream(data + k) : T(1);
            const bool zero = ok && v == T(0);
            if (binarize) v = v != T(0) ? T(1) : T(0);
            if (ok) {
                atomicAdd(col_sum + c, v);
                acc += v;
            }
            int p = __shfl_up_sync(0xffffffffu, c, 1);
            const int last = __shfl_sync(0xffffffffu, c, 31);
            if (lane == 0) p = carry;
            carry = last;
            bad |= (ok && c <= p) | (zero << 1);
        }
        acc = warp_sum(acc);
        if (lane == 0) row_sum[row] = acc;
    }
    if (status != nullptr && bad) atomicOr(status, bad);
}

// ---- tiled reduce (fp32, rows with sorted column indices) -----------------------------------------------
// The kernel above issues one global RED per non-zero into the D-vector of column sums: 6e9 atomics at
// BASELINE configs[1], and it is their rate (not HBM) that bounds it.  Here a CTA
// owns a block of kTileRows rows and sweeps the column range tile by tile (kTileCols columns): the tile's
// column sums AND entry counts live in shared memory, every non-zero costs two shared-memory atomics, and the
// tile is flushed to global memory once per (row block, tile) -- ~30x fewer global atomics.  Rows are sorted, so
// the entries of a row that fall in a tile are one contiguous segment; a per-row cursor in shared memory marks
// where the next tile continues (no searching).  By-products, for free:
//   * the entry count per (row chunk, column): exactly the histogram the CSR transposition needs
//     (transpose.cu::transpose_count_kernel, one more pass of 6e9 global atomics otherwise),
//   * the same canonical-form verdict: strictly increasing indices (bit0), explicit zeros (bit1).
constexpr int kTileCols = 12288;   // 2 x 48 KB of shared memory per CTA -> 2 CTAs per SM
constexpr int kTileRows = 512;
constexpr int kTileThreads = 512;

template <bool binarize>
__global__ void __launch_bounds__(kTileThreads, 2)
tfidf_reduce_tiled_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                          const float* __restrict__ data, int64_t n_rows, int32_t n_cols, float* __restrict__ row_sum,
                          float* __restrict__ col_sum, int* __restrict__ status, int32_t* __restrict__ col_count,
                          const int64_t* __restrict__ chunk_bounds, int32_t n_chunks, int64_t row_base,
                          uint16_t* __restrict__ rb_count) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* sums = reinterpret_cast<float*>(smem_raw);
    unsigned* cnts = reinterpret_cast<unsigned*>(smem_raw + sizeof(float) * kTileCols);
    int* cur = reinterpret_cast<int*>(smem_raw + 2 * sizeof(float) * kTileCols);      // offset into the row
    float* rsum = reinterpret_cast<float*>(cur + kTileRows);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    constexpr int kWarps = kTileThreads / 32;
    const int64_t r0 = (int64_t)blockIdx.x * kTileRows;
    const int rows_here = (int)((n_rows - r0) < kTileRows ? (n_rows - r0) : kTileRows);
    for (int r = threadIdx.x; r < kTileRows; r += kTileThreads) {
        cur[r] = 0;
        rsum[r] = 0.f;
    }
    // row chunk of this block (chunk bounds are multiples of kTileRows in absolute row numbers)
    int chunk = 0;
    if (col_count != nullptr) {
        const int64_t abs_row = row_base + r0;
        for (int c = 1; c < n_chunks; ++c) chunk += (abs_row >= chunk_bounds[c]) ? 1 : 0;
    }
    int bad = 0;
    const int n_tiles = (n_cols + kTileCols - 1) / kTileCols;
    for (int t = 0; t < n_tiles; ++t) {
        const int c_lo = t * kTileCols;
        const int c_hi = (c_lo + kTileCols < n_cols) ? c_lo + kTileCols : n_cols;
        for (int j = threadIdx.x; j < kTileCols; j += kTileThreads) {
            sums[j] = 0.f;
            cnts[j] = 0u;
        }
        __syncthreads();
        for (int r = warp; r < rows_here; r += kWarps) {
            const int64_t s0 = __ldg(indptr + r0 + r), e = __ldg(indptr + r0 + r + 1);
            int64_t k = s0 + cur[r];
            float acc = 0.f;
            int prev_last = c_lo - 1;          // last column index seen in this tile's segment
            for (;;) {
                // three 32-wide segments in flight per lane
                const int64_t k0 = k + lane, k1 = k0 + 32, k2 = k0 + 64;
                const int c0 = k0 < e ? ld_stream(indices + k0) : 0x7fffffff;
                const int c1 = k1 < e ? ld_stream(indices + k1) : 0x7fffffff;
                const int c2 = k2 < e ? ld_stream(indices + k2) : 0x7fffffff;
                float v0 = k0 < e ? ld_stream(data + k0) : 1.f;
                float v1 = k1 < e ? ld_stream(data + k1) : 1.f;
                float v2 = k2 < e ? ld_stream(data + k2) : 1.f;
                int taken = 0;
                bool stop = false;
#pragma unroll
                for (int u = 0; u < 3; ++u) {
                    const int c = u == 0 ? c0 : (u == 1 ? c1 : c2);
                    float v = u == 0 ? v0 : (u == 1 ? v1 : v2);
                    const bool in = !stop && c < c_hi;             // warp-uniform `stop`, per-lane `c`
                    const unsigned m = __ballot_sync(0xffffffffu, in);
                    // entries of the tile form a prefix of the segment iff the row is sorted
                    const int n_in = __popc(m);
                    const bool prefix = (m == (n_in == 32 ? 0xffffffffu : ((1u << n_in) - 1u)));
                    int p = __shfl_up_sync(0xffffffffu, c, 1);
                    if (lane == 0) p = prev_last;
                    if (in) {
                        bad |= (c <= p) | (c < c_lo) | ((v == 0.f) << 1);
                        if (binarize) v = v != 0.f ? 1.f : 0.f;
                        if (c >= c_lo) {
                            atomicAdd(&sums[c - c_lo], v);
                            atomicAdd(&cnts[c - c_lo], 1u);
                        }
                        acc += v;
                    }
                    bad |= prefix ? 0 : 1;
                    if (n_in > 0) prev_last = __shfl_sync(0xffffffffu, c, n_in - 1);
                    taken += n_in;
                    if (n_in < 32) stop = true;
                }
                k += taken;
                if (stop || k >= e) break;
            }
            acc = warp_sum(acc);
            __syncwarp();      // every lane has read cur[r] (racecheck: intra-warp write-after-read without this)
            if (lane == 0) {
                cur[r] = (int)(k - s0);
                rsum[r] += acc;
                if (t == n_tiles - 1 && k != e) bad |= 1;     // left-over entries: index >= n_cols or unsorted
            }
        }
        __syncthreads();
        for (int j = threadIdx.x; j < c_hi - c_lo; j += kTileThreads) {
            const unsigned cn = cnts[j];
            if (cn != 0u) {
                atomicAdd(col_sum + c_lo + j, sums[j]);
                if (col_count != nullptr) atomicAdd(col_count + (size_t)chunk * n_cols + c_lo + j, (int)cn);
            }
            // entries of this ROW BLOCK per column (<= kTileRows, fits 16 bits): the tiled transposition derives
            // every block's write offsets from these, so it needs no global atomics (transpose.cu)
            if (rb_count != nullptr) rb_count[((size_t)(row_base / kTileRows) + blockIdx.x) * n_cols + c_lo + j] = (uint16_t)cn;
        }
        __syncthreads();
    }
    for (int r = threadIdx.x; r < rows_here; r += kTileThreads) row_sum[r0 + r] = rsum[r];
    if (status != nullptr && bad) atomicOr(status, bad);
}

template <typename T>
__global__ void tfidf_idf_kernel(const T* __restrict__ col_sum, int32_t n_cols, T n_obs, uint32_t flags,
                                 T* __restrict__ idf) {
    int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_cols) return;
    T v = n_obs / col_sum[j];  // IEEE division; empty column -> inf, never gathered (App. A.4)
    if (flags & MUB_TFIDF_LOG_IDF) v = log1p(v);
    idf[j] = v;
}

template <typename T>
__device__ __forceinline__ T tfidf_value(T c, T inv_r, T idf, T sf, uint32_t flags) {
    // association order of the reference: ((1/r) * c) * sf -> log1p -> * idf -> log1p
    if (flags & MUB_TFIDF_BINARIZE) c = (c != T(0)) ? T(1) : T(0);   // binarize() fused (preproc.py:149)
    T t;
    if constexpr (sizeof(T) == 4) {
        t = __fmul_rn(inv_r, c);
        if (!(flags & MUB_TFIDF_NO_SCALE)) t = __fmul_rn(t, sf);
        if (flags & MUB_TFIDF_LOG_TF) t = log1pf(t);
        t = __fmul_rn(t, idf);
        if (flags & MUB_TFIDF_LOG_TFIDF) t = log1pf(t);
    } else {
        t = __dmul_rn(inv_r, c);
        if (!(flags & MUB_TFIDF_NO_SCALE)) t = __dmul_rn(t, sf);
        if (flags & MUB_TFIDF_LOG_TF) t = log1p(t);
        t = __dmul_rn(t, idf);
        if (flags & MUB_TFIDF_LOG_TFIDF) t = log1p(t);
    }
    // inf * 0 on all-explicit-zero rows: the reference intends 0 there (preproc.py:119)
    return (t != t) ? T(0) : t;
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
tfidf_apply_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                   const T* data_in, T* data_out, int64_t n_rows, const T* __restrict__ row_sum,
                   const T* __restrict__ idf, T sf, uint32_t flags) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (int64_t)blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5);
    const int64_t n_warps = (int64_t)gridDim.x * kWarpsPerCta;
    for (int64_t row = warp; row < n_rows; row += n_warps) {
        const int64_t start = __ldg(indptr + row), end = __ldg(indptr + row + 1);
        if (start == end) continue;
        const T inv_r = T(1) / __ldg(row_sum + row);  // 1.0 / n_peaks, preproc.py:94
        int64_t k = start + lane;
        for (; k + 96 < end; k += 128) {
            int c0 = ld_stream(indices + k), c1 = ld_stream(indices + k + 32);
            int c2 = ld_stream(indices + k + 64), c3 = ld_stream(indices + k + 96);
            T v0 = ld_stream_rw(data_in + k), v1 = ld_stream_rw(data_in + k + 32);
            T v2 = ld_stream_rw(data_in + k + 64), v3 = ld_stream_rw(data_in + k + 96);
            T i0 = __ldg(idf + c0), i1 = __ldg(idf + c1), i2 = __ldg(idf + c2), i3 = __ldg(idf + c3);
            st_stream(data_out + k, tfidf_value(v0, inv_r, i0, sf, flags));
            st_stream(data_out + k + 32, tfidf_value(v1, inv_r, i1, sf, flags));
            st_stream(data_out + k + 64, tfidf_value(v2, inv_r, i2, sf, flags));
            st_stream(data_out + k + 96, tfidf_value(v3, inv_r, i3, sf, flags));
        }
        for (; k < end; k += 32) {
            int c = ld_stream(indices + k);
            T v = ld_stream_rw(data_in + k);
            st_stream(data_out + k, tfidf_value(v, inv_r, __ldg(idf + c), sf, flags));
        }
    }
}

static int grid_for_rows(int64_t n_rows) {
    // persistent-style: 8 CTAs of 256 threads per SM (full occupancy), never more warps than rows
    int64_t want = (n_rows + kWarpsPerCta - 1) / kWarpsPerCta;
    int64_t cap = (int64_t)sm_count() * 8;
    int64_t g = want < cap ? want : cap;
    return (int)(g < 1 ? 1 : g);
}

template <typename T>
int tfidf_reduce(const int64_t* indptr, const int32_t* indices, const T* data, int64_t n_rows,
                 int32_t n_cols, T* row_sum, T* col_sum, int* status, uint32_t flags, mub_stream_t stream) {
    MUB_REQUIRE(n_rows >= 0 && n_cols >= 0, "tfidf_reduce: negative shape");
    if (n_rows == 0) return 0;
    MUB_REQUIRE(indptr && row_sum && col_sum, "tfidf_reduce: null pointer");
    if (flags & MUB_TFIDF_BINARIZE)
        tfidf_reduce_kernel<T, true><<<grid_for_rows(n_rows), kThreads, 0, (cudaStream_t)stream>>>(
            indptr, indices, data, n_rows, row_sum, col_sum, status);
    else
        tfidf_reduce_kernel<T, false><<<grid_for_rows(n_rows), kThreads, 0, (cudaStream_t)stream>>>(
            indptr, indices, data, n_rows, row_sum, col_sum, status);
    return check_launch("tfidf_reduce");
}

template <typename T>
int tfidf_idf(const T* col_sum, int32_t n_cols, double n_obs, uint32_t flags, T* idf, mub_stream_t stream) {
    MUB_REQUIRE(n_cols >= 0, "tfidf_idf: negative n_cols");
    if (n_cols == 0) return 0;
    tfidf_idf_kernel<T><<<(n_cols + 255) / 256, 256, 0, (cudaStream_t)stream>>>(col_sum, n_cols, (T)n_obs,
                                                                              flags, idf);
    return check_launch("tfidf_idf");
}

template <typename T>
int tfidf_apply(const int64_t* indptr, const int32_t* indices, const T* data_in, T* data_out,
                int64_t n_rows, int32_t n_cols, const T* row_sum, const T* idf, T sf, uint32_t flags,
                mub_stream_t stream) {
    MUB_REQUIRE(n_rows >= 0 && n_cols >= 0, "tfidf_apply: negative shape");
    MUB_REQUIRE(!((flags & MUB_TFIDF_LOG_TFIDF) && (flags & (MUB_TFIDF_LOG_TF | MUB_TFIDF_LOG_IDF))),
                "tfidf_apply: LOG_TFIDF excludes LOG_TF/LOG_IDF (preproc.py:69-73)");
    if (n_rows == 0) return 0;
    tfidf_apply_kernel<T><<<grid_for_rows(n_rows), kThreads, 0, (cudaStream_t)stream>>>(
        indptr, indices, data_in, data_out, n_rows, row_sum, idf, sf, flags);
    return check_launch("tfidf_apply");
}

static size_t tiled_smem_bytes() { return 2 * sizeof(float) * kTileCols + 2 * sizeof(int) * kTileRows; }

}  // namespace mub

extern "C" {

int mub_tfidf_reduce_tiled_f32(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_rows,
                               int32_t n_cols, float* row_sum, float* col_sum, int32_t* status, uint32_t flags,
                               int32_t* col_count, const int64_t* chunk_bounds, int32_t n_chunks, int64_t row_base,
                               uint16_t* rb_count, mub_stream_t stream) {
    MUB_REQUIRE(n_rows >= 0 && n_cols >= 0, "tfidf_reduce_tiled: negative shape");
    if (n_rows == 0) return 0;
    MUB_REQUIRE(indptr && row_sum && col_sum && status, "tfidf_reduce_tiled: null pointer (status is mandatory: it reports rows "
                "that are not sorted, for which the result is invalid)");
    MUB_REQUIRE(col_count == nullptr || (chunk_bounds != nullptr && n_chunks >= 1), "tfidf_reduce_tiled: counts need chunk bounds");
    MUB_REQUIRE((row_base % mub::kTileRows) == 0, "tfidf_reduce_tiled: row_base must be a multiple of %d", mub::kTileRows);
    const size_t smem = mub::tiled_smem_bytes();
    const int64_t grid = (n_rows + mub::kTileRows - 1) / mub::kTileRows;
    MUB_REQUIRE(grid < (1ll << 31), "tfidf_reduce_tiled: too many rows");
    cudaStream_t s = (cudaStream_t)stream;
    if (flags & MUB_TFIDF_BINARIZE) {
        cudaFuncSetAttribute(mub::tfidf_reduce_tiled_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        mub::tfidf_reduce_tiled_kernel<true><<<(int)grid, mub::kTileThreads, smem, s>>>(
            indptr, indices, data, n_rows, n_cols, row_sum, col_sum, status, col_count, chunk_bounds, n_chunks, row_base, rb_count);
    } else {
        cudaFuncSetAttribute(mub::tfidf_reduce_tiled_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        mub::tfidf_reduce_tiled_kernel<false><<<(int)grid, mub::kTileThreads, smem, s>>>(
            indptr, indices, data, n_rows, n_cols, row_sum, col_sum, status, col_count, chunk_bounds, n_chunks, row_base, rb_count);
    }
    return mub::check_launch("tfidf_reduce_tiled");
}

int mub_tfidf_tile_rows(void) { return mub::kTileRows; }

int mub_tfidf_reduce_f32(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_rows,
                         int32_t n_cols, float* row_sum, float* col_sum, int32_t* status, uint32_t flags,
                         mub_stream_t stream) {
    return mub::tfidf_reduce<float>(indptr, indices, data, n_rows, n_cols, row_sum, col_sum, status, flags, stream);
}
int mub_tfidf_reduce_f64(const int64_t* indptr, const int32_t* indices, const double* data, int64_t n_rows,
                         int32_t n_cols, double* row_sum, double* col_sum, int32_t* status, uint32_t flags,
                         mub_stream_t stream) {
    return mub::tfidf_reduce<double>(indptr, indices, data, n_rows, n_cols, row_sum, col_sum, status, flags, stream);
}
int mub_tfidf_idf_f32(const float* col_sum, int32_t n_cols, double n_obs_total, uint32_t flags, float* idf,
                      mub_stream_t stream) {
    return mub::tfidf_idf<float>(col_sum, n_cols, n_obs_total, flags, idf, stream);
}
int mub_tfidf_idf_f64(const double* col_sum, int32_t n_cols, double n_obs_total, uint32_t flags, double* idf,
                      mub_stream_t stream) {
    return mub::tfidf_idf<double>(col_sum, n_cols, n_obs_total, flags, idf, stream);
}
int mub_tfidf_apply_f32(const int64_t* indptr, const int32_t* indices, const float* data_in, float* data_out,
                        int64_t n_rows, int32_t n_cols, const float* row_sum, const float* idf,
                        float scale_factor, uint32_t flags, mub_stream_t stream) {
    return mub::tfidf_apply<float>(indptr, indices, data_in, data_out, n_rows, n_cols, row_sum, idf,
                                   scale_factor, flags, stream);
}
int mub_tfidf_apply_f64(const int64_t* indptr, const int32_t* indices, const double* data_in,
                        double* data_out, int64_t n_rows, int32_t n_cols, const double* row_sum,
                        const double* idf, double scale_factor, uint32_t flags, mub_stream_t stream) {
    return mub::tfidf_apply<double>(indptr, indices, data_in, data_out, n_rows, n_cols, row_sum, idf,
                                    scale_factor, flags, stream);
}

}  // extern "C"
