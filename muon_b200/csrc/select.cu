// Row-and-column selection of a CSR: out = A[rows][:, kept columns], the kept columns renumbered.  This is how a
// device-resident MOFA view is cut into (view, group) blocks and restricted to its use_var features without leaving
// the GPU (the host path does the same with scipy fancy indexing).
//
// count : warp per output row; with a column map every lane looks up one entry of a 32-wide chunk, a ballot counts
//         the kept ones.  Without one the count is the source row's length (one thread per row).
// fill  : warp per output row; each 32-entry chunk is compacted with __ballot_sync / __popc, so the kept entries keep
//         their order.  The next chunk's loads are issued before the current chunk is stored.  Stores never leave the
//         output row's range [out_indptr[i], out_indptr[i+1]).
//
// indptr values are absolute offsets into indices / data (a view may start anywhere in larger arrays, beyond 2^31).
#include "common.cuh"

namespace mub {

constexpr int kSelThreads = 256;
constexpr int kSelWarps = kSelThreads / 32;

__device__ __forceinline__ int64_t source_row(const int64_t* rows, int64_t i) { return rows ? __ldg(rows + i) : i; }

// column of a source index after the map: -1 = dropped (also for an index outside [0, n_cols))
__device__ __forceinline__ int mapped(const int32_t* __restrict__ col_map, int32_t n_cols, int c) {
    return (unsigned)c < (unsigned)n_cols ? __ldg(col_map + c) : -1;
}

__global__ void __launch_bounds__(kSelThreads)
select_count_rows_kernel(const int64_t* __restrict__ indptr, const int64_t* __restrict__ rows, int64_t n_rows_out,
                         int64_t* __restrict__ out_len) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_rows_out; i += stride) {
        const int64_t r = source_row(rows, i);
        out_len[i] = __ldg(indptr + r + 1) - __ldg(indptr + r);
    }
}

__global__ void __launch_bounds__(kSelThreads)
select_count_mapped_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices, int32_t n_cols,
                           const int64_t* __restrict__ rows, int64_t n_rows_out, const int32_t* __restrict__ col_map,
                           int64_t* __restrict__ out_len) {
    const int lane = threadIdx.x & 31;
    const int64_t n_warps = (int64_t)gridDim.x * kSelWarps;
    for (int64_t i = (int64_t)blockIdx.x * kSelWarps + (threadIdx.x >> 5); i < n_rows_out; i += n_warps) {
        const int64_t r = source_row(rows, i);
        const int64_t s = __ldg(indptr + r), e = __ldg(indptr + r + 1);
        int64_t kept = 0;
        // two chunks in flight per lane
        for (int64_t k = s + lane; k - lane < e; k += 64) {
            const int c0 = k < e ? ld_stream(indices + k) : -1;
            const int c1 = k + 32 < e ? ld_stream(indices + k + 32) : -1;
            const bool in0 = c0 >= 0 && mapped(col_map, n_cols, c0) >= 0;
            const bool in1 = c1 >= 0 && mapped(col_map, n_cols, c1) >= 0;
            kept += __popc(__ballot_sync(0xffffffffu, in0)) + __popc(__ballot_sync(0xffffffffu, in1));
        }
        if (lane == 0) out_len[i] = kept;
    }
}

__global__ void __launch_bounds__(kSelThreads)
select_fill_rows_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                        const float* __restrict__ data, const int64_t* __restrict__ rows, int64_t n_rows_out,
                        const int64_t* __restrict__ out_indptr, int32_t* __restrict__ out_indices,
                        float* __restrict__ out_data) {
    const int lane = threadIdx.x & 31;
    const int64_t n_warps = (int64_t)gridDim.x * kSelWarps;
    for (int64_t i = (int64_t)blockIdx.x * kSelWarps + (threadIdx.x >> 5); i < n_rows_out; i += n_warps) {
        const int64_t o = __ldg(out_indptr + i), n = __ldg(out_indptr + i + 1) - o;
        if (n <= 0) continue;
        const int64_t s = __ldg(indptr + source_row(rows, i));
        // four chunks of loads in flight per lane before the first store
        int64_t k = lane;
        for (; k + 96 < n; k += 128) {
            const int c0 = ld_stream(indices + s + k), c1 = ld_stream(indices + s + k + 32);
            const int c2 = ld_stream(indices + s + k + 64), c3 = ld_stream(indices + s + k + 96);
            const float v0 = ld_stream(data + s + k), v1 = ld_stream(data + s + k + 32);
            const float v2 = ld_stream(data + s + k + 64), v3 = ld_stream(data + s + k + 96);
            out_indices[o + k] = c0; out_indices[o + k + 32] = c1; out_indices[o + k + 64] = c2; out_indices[o + k + 96] = c3;
            out_data[o + k] = v0; out_data[o + k + 32] = v1; out_data[o + k + 64] = v2; out_data[o + k + 96] = v3;
        }
        for (; k < n; k += 32) {
            out_indices[o + k] = ld_stream(indices + s + k);
            out_data[o + k] = ld_stream(data + s + k);
        }
    }
}

__global__ void __launch_bounds__(kSelThreads)
select_fill_mapped_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                          const float* __restrict__ data, int32_t n_cols, const int64_t* __restrict__ rows,
                          int64_t n_rows_out, const int32_t* __restrict__ col_map, const int64_t* __restrict__ out_indptr,
                          int32_t* __restrict__ out_indices, float* __restrict__ out_data) {
    const int lane = threadIdx.x & 31;
    const unsigned below = (1u << lane) - 1u;
    const int64_t n_warps = (int64_t)gridDim.x * kSelWarps;
    for (int64_t i = (int64_t)blockIdx.x * kSelWarps + (threadIdx.x >> 5); i < n_rows_out; i += n_warps) {
        int64_t o = __ldg(out_indptr + i);
        const int64_t o_end = __ldg(out_indptr + i + 1);
        if (o_end <= o) continue;                          // nothing kept (or an empty row): the source is not read
        const int64_t r = source_row(rows, i);
        const int64_t s = __ldg(indptr + r), e = __ldg(indptr + r + 1);
        int64_t k = s + lane;
        int c = k < e ? ld_stream(indices + k) : -1;
        float v = k < e ? ld_stream(data + k) : 0.f;
        while (k - lane < e) {
            // next chunk's loads first, then the current chunk's map lookups and stores
            const int64_t kn = k + 32;
            const int cn = kn < e ? ld_stream(indices + kn) : -1;
            const float vn = kn < e ? ld_stream(data + kn) : 0.f;
            const int m = c >= 0 ? mapped(col_map, n_cols, c) : -1;
            const unsigned ball = __ballot_sync(0xffffffffu, m >= 0);
            const int64_t p = o + __popc(ball & below);
            if (m >= 0 && p < o_end) {
                out_indices[p] = m;
                out_data[p] = v;
            }
            o += __popc(ball);
            k = kn;
            c = cn;
            v = vn;
        }
    }
}

inline int select_grid(int64_t n_items_per_cta_units) {
    const int64_t cap = (int64_t)sm_count() * 16;
    const int64_t g = n_items_per_cta_units < cap ? n_items_per_cta_units : cap;
    return (int)(g < 1 ? 1 : g);
}

}  // namespace mub

extern "C" {

int mub_csr_select_count(const int64_t* indptr, const int32_t* indices, int64_t n_rows_src, int32_t n_cols_src,
                         const int64_t* rows, int64_t n_rows_out, const int32_t* col_map, int64_t* out_len,
                         mub_stream_t stream) {
    MUB_REQUIRE(n_rows_src >= 0 && n_cols_src >= 0 && n_rows_out >= 0, "csr_select_count: negative shape");
    MUB_REQUIRE(rows != nullptr || n_rows_out == n_rows_src,
                "csr_select_count: rows = NULL selects every row, so n_rows_out must equal n_rows_src");
    if (n_rows_out == 0) return 0;
    MUB_REQUIRE(n_rows_src > 0, "csr_select_count: rows selected from a matrix without rows");
    MUB_REQUIRE(indptr && out_len, "csr_select_count: null pointer");
    MUB_REQUIRE(col_map == nullptr || indices != nullptr, "csr_select_count: a column map needs the indices");
    cudaStream_t s = (cudaStream_t)stream;
    if (col_map == nullptr) {
        mub::select_count_rows_kernel<<<mub::select_grid((n_rows_out + mub::kSelThreads - 1) / mub::kSelThreads),
                                        mub::kSelThreads, 0, s>>>(indptr, rows, n_rows_out, out_len);
    } else {
        mub::select_count_mapped_kernel<<<mub::select_grid((n_rows_out + mub::kSelWarps - 1) / mub::kSelWarps),
                                          mub::kSelThreads, 0, s>>>(indptr, indices, n_cols_src, rows, n_rows_out,
                                                                    col_map, out_len);
    }
    return mub::check_launch("csr_select_count");
}

int mub_csr_select_fill_f32(const int64_t* indptr, const int32_t* indices, const float* data, int32_t n_cols_src,
                            const int64_t* rows, int64_t n_rows_out, const int32_t* col_map, const int64_t* out_indptr,
                            int32_t* out_indices, float* out_data, mub_stream_t stream) {
    MUB_REQUIRE(n_cols_src >= 0 && n_rows_out >= 0, "csr_select_fill: negative shape");
    if (n_rows_out == 0) return 0;
    MUB_REQUIRE(indptr && indices && data && out_indptr, "csr_select_fill: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    const int grid = mub::select_grid((n_rows_out + mub::kSelWarps - 1) / mub::kSelWarps);
    if (col_map == nullptr)
        mub::select_fill_rows_kernel<<<grid, mub::kSelThreads, 0, s>>>(indptr, indices, data, rows, n_rows_out, out_indptr,
                                                                      out_indices, out_data);
    else
        mub::select_fill_mapped_kernel<<<grid, mub::kSelThreads, 0, s>>>(indptr, indices, data, n_cols_src, rows,
                                                                        n_rows_out, col_map, out_indptr, out_indices,
                                                                        out_data);
    return mub::check_launch("csr_select_fill");
}

}  // extern "C"
