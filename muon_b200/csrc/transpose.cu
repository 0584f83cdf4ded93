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

// PAIRS: (row, value) is written as ONE 8-byte pair (int2, in t_indices; t_data unused) instead of into two arrays:
// one scattered store per non-zero instead of two (the fill is bound by the rate of scattered L2 operations, not by
// bytes).
template <bool PAIRS, typename V>
__device__ __forceinline__ void store_entry(int32_t* __restrict__ t_indices, V* __restrict__ t_data,
                                            unsigned long long slot, int32_t r, V v) {
    if constexpr (PAIRS) {
        static_assert(sizeof(V) == 4, "pairs hold float32 values");
        reinterpret_cast<int2*>(t_indices)[slot] = make_int2(r, __float_as_int(v));
    } else {
        t_indices[slot] = r;
        t_data[slot] = v;
    }
}

template <bool PAIRS, typename V>
__global__ void __launch_bounds__(256)
transpose_fill_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                      const V* __restrict__ data, int64_t n_rows, int64_t row_offset,
                      unsigned long long* cursor, int32_t* __restrict__ t_indices, V* __restrict__ t_data) {
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
            const V v0 = ld_stream(data + k), v1 = ld_stream(data + k + 32);
            const V v2 = ld_stream(data + k + 64), v3 = ld_stream(data + k + 96);
            const unsigned long long s0 = atomicAdd(cursor + c0, 1ull), s1 = atomicAdd(cursor + c1, 1ull);
            const unsigned long long s2 = atomicAdd(cursor + c2, 1ull), s3 = atomicAdd(cursor + c3, 1ull);
            store_entry<PAIRS>(t_indices, t_data, s0, r, v0);
            store_entry<PAIRS>(t_indices, t_data, s1, r, v1);
            store_entry<PAIRS>(t_indices, t_data, s2, r, v2);
            store_entry<PAIRS>(t_indices, t_data, s3, r, v3);
        }
        for (; k < e; k += 32) {
            const int c = ld_stream(indices + k);
            const V v = ld_stream(data + k);
            store_entry<PAIRS>(t_indices, t_data, atomicAdd(cursor + c, 1ull), r, v);
        }
    }
}

// the two atomic-cursor entry points: shared validation, cursors seeded from the scanned histogram, one warp per row
template <bool PAIRS, typename V>
static int launch_transpose_fill(const char* name, const int64_t* indptr, const int32_t* indices, const V* data,
                                 int64_t n_rows, int32_t n_cols, int64_t row_offset, const int64_t* t_indptr,
                                 int64_t* cursor, int32_t* t_indices, V* t_data, mub_stream_t stream) {
    MUB_REQUIRE(n_rows >= 0 && n_cols >= 0, "%s: negative shape", name);
    if (n_rows == 0 || n_cols == 0) return 0;
    MUB_REQUIRE(indptr && t_indptr && cursor && t_indices && (PAIRS || t_data), "%s: null pointer", name);
    MUB_REQUIRE(!PAIRS || ((uintptr_t)t_indices & 7) == 0, "%s: t_pairs must be 8-byte aligned", name);
    cudaStream_t s = (cudaStream_t)stream;
    copy_i64_kernel<<<(n_cols + 255) / 256, 256, 0, s>>>(t_indptr, cursor, n_cols);
    int64_t want = (n_rows + 7) / 8;
    int64_t cap = (int64_t)sm_count() * 8;
    int grid = (int)(want < cap ? want : cap);
    if (grid < 1) grid = 1;
    transpose_fill_kernel<PAIRS, V><<<grid, 256, 0, s>>>(indptr, indices, data, n_rows, row_offset,
                                                     (unsigned long long*)cursor, t_indices, t_data);
    return check_launch(name);
}

// ---- tiled fill: no global atomics, deterministic ------------------------------------------------------------
// The atomic-cursor fill above spends one global ATOM (with return) plus one scattered 8-byte store per non-zero,
// and the order in which slots are claimed -- hence the order of the entries inside a transposed row, hence the fp32
// summation order of every A^T Y product -- changes from run to run.  When the TF-IDF reduce pass has left the
// entry count of every (512-row block, column) behind (tfidf.cu, rb_count), the write offset of block b in column c
// is  t_indptr[c] + sum of the counts of the panel's earlier blocks  -- a column-wise scan.  Inside its block a CTA
// sweeps the columns tile by tile; warp w owns the 32 consecutive rows [32w, 32w + 32) and walks them in order.
// Per tile it first counts its entries per column, the counts are scanned over the warps in warp order, and a second
// walk places every entry at the next slot of its (warp, column) cursor.  Every transposed row therefore lists its
// cells in ascending order, on every run.
//
// The block's slots of one column are consecutive: ~15 pairs (120 B) at 3 % density.  Written straight from the
// walk, every lane of a warp store hits a different transposed row, so each non-zero costs an L2 write of its own,
// and those writes, not the reads, bound the fill.  So the second walk places the tile's entries in shared memory,
// ordered by (column, row), and the CTA then copies every (block, column) run out with consecutive lanes.  A tile
// with more entries than the staging area holds (a dense stretch of columns) writes them straight to global memory
// instead; the slots, hence the result, are the same.
//
// Loads: lane l of warp w keeps the cursor of row 32w + l in a register, and a warp issues the loads of kFillGroup
// rows before it consumes any of them (the row starts and cursors are known, so no load waits on another).  The first
// walk records how many entries of each row fall inside the tile, so the second walk loads exactly those.  A CTA sweeps
// one slab of column tiles of its row block (blockIdx.y); the slab's first cursor of every row is found by a binary
// search of the sorted row.  Slabs give every launch enough CTAs to keep two per SM busy.
constexpr int kFillTileCols = 512;     // one column of the tile per thread in the scans
constexpr int kFillRows = 512;         // must equal the reduce kernel's block height (mub_tfidf_tile_rows)
constexpr int kFillThreads = 512;
constexpr int kFillWarps = kFillThreads / 32;
constexpr int kFillRowsPerWarp = kFillRows / kFillWarps;
static_assert(kFillRowsPerWarp == 32, "lane l of a warp holds the cursor of the warp's row l");
static_assert(kFillTileCols == kFillThreads, "thread j scans column j of the tile");
constexpr int kFillGroup = 16;         // rows of a warp whose (index, value) loads are in flight together in the
                                       // placing walk; the counting walk loads the indices of all 32 rows at once
                                       // (~15 entries per row and tile at 3 % density: one 32-wide load each, longer
                                       // segments continue)
constexpr int kFillStage = 11776;      // staged pairs per tile: 1.5x the ~7.9k of a 512 x 512 tile at 3 % density
static_assert((sizeof(int2) * kFillStage) % 16 == 0 && (sizeof(uint16_t) * kFillWarps * kFillTileCols) % 16 == 0,
              "the cursors follow the staging area and are cleared with 16-byte stores");
// staging + column starts + per-column write offsets + 16-bit per-warp cursors: 112 KB, two CTAs per SM
constexpr size_t kFillSmem = sizeof(int2) * kFillStage + sizeof(uint32_t) * (2 * kFillTileCols + 1) +
                             sizeof(uint16_t) * kFillWarps * kFillTileCols;

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

// Besides the pairs, the kernel checks the pattern against the counts it was given: a (block, column) whose entries
// differ from rb_count, or a row that is not sorted or holds a column >= n_cols, sets bit0 of status.  Slots at or
// past t_indptr[n_cols] or the panel's non-zero count are never written, so a matrix modified after its counts were
// taken cannot corrupt memory.
__global__ void __launch_bounds__(kFillThreads, 2)
transpose_fill_tiled_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                            const float* __restrict__ data, int64_t n_rows, int32_t n_cols, int tiles_per_slab,
                            const uint16_t* __restrict__ rb_count, const uint32_t* __restrict__ base,
                            const int64_t* __restrict__ t_indptr, int2* __restrict__ t_pairs, int* __restrict__ status) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    // 16-byte aligned first: the staging area and the cursors (cleared with 16-byte stores)
    int2* stage = reinterpret_cast<int2*>(smem_raw);                                 // [kFillStage] (column, row) order
    uint16_t* wcur = reinterpret_cast<uint16_t*>(stage + kFillStage);                // [kFillWarps][kFillTileCols]
    uint32_t* cstart = reinterpret_cast<uint32_t*>(wcur + kFillWarps * kFillTileCols);   // [kFillTileCols + 1] into stage
    uint32_t* cbase = cstart + kFillTileCols + 1;                                    // [kFillTileCols] block's slot
    __shared__ uint32_t wsum[kFillWarps];
    constexpr unsigned kAll = 0xffffffffu;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t r0 = (int64_t)blockIdx.x * kFillRows;
    const int64_t row0 = r0 + warp * kFillRowsPerWarp;                              // the warp's first row
    const int n_tiles = (n_cols + kFillTileCols - 1) / kFillTileCols;
    const int t0 = blockIdx.y * tiles_per_slab;
    const int t1 = (t0 + tiles_per_slab < n_tiles) ? t0 + tiles_per_slab : n_tiles;
    // slots that exist: the entries the counts announce, and no more than the panel holds (the size of t_pairs)
    const int64_t held = __ldg(indptr + n_rows) - __ldg(indptr), announced = __ldg(t_indptr + n_cols);
    const unsigned long long total = (unsigned long long)(announced < held ? announced : held);
    // lane l: row row0 + l -- its first non-zero and its length
    int64_t rs = 0;
    int len = 0;
    if (row0 + lane < n_rows) {
        rs = __ldg(indptr + row0 + lane);
        len = (int)(__ldg(indptr + row0 + lane + 1) - rs);
    }
    int cur = 0;
    if (t0 > 0) {              // first entry of the slab: lower bound of its first column in the sorted row
        const int c_first = t0 * kFillTileCols;
        int hi = len;
        while (cur < hi) {
            const int mid = (int)(((unsigned)cur + (unsigned)hi) >> 1);
            if (__ldg(indices + rs + mid) < c_first) cur = mid + 1;
            else hi = mid;
        }
    }
    int64_t rk = rs + cur;     // lane l: next entry of its row ...
    int rem = len - cur;       // ... and the entries left in it
    int bad = 0;
    uint16_t* my_cur = wcur + warp * kFillTileCols;
    uint32_t* my_cur2 = reinterpret_cast<uint32_t*>(my_cur);   // two 16-bit counters per word for the counting atomics
    const uint32_t* blk_base = base + (size_t)blockIdx.x * n_cols;
    const uint16_t* blk_count = rb_count + (size_t)blockIdx.x * n_cols;
    constexpr int kCurVecs = kFillWarps * kFillTileCols * (int)sizeof(uint16_t) / 16;
    for (int j = threadIdx.x; j < kCurVecs; j += kFillThreads) reinterpret_cast<uint4*>(wcur)[j] = make_uint4(0u, 0u, 0u, 0u);
    __syncthreads();
    for (int t = t0; t < t1; ++t) {
        const int c_lo = t * kFillTileCols;
        const int c_hi = (c_lo + kFillTileCols < n_cols) ? c_lo + kFillTileCols : n_cols;
        // thread j's operands of the scan below (column c_lo + j), in flight during the first walk
        const bool col_in = c_lo + (int)threadIdx.x < c_hi;
        const uint32_t want = col_in ? (uint32_t)__ldg(blk_count + c_lo + threadIdx.x) : 0u;
        const uint32_t slot0 = col_in ? __ldg(blk_base + c_lo + threadIdx.x) : 0u;
        // walk 1: entries per (warp, column) of this tile, and per row (lane) the number of its entries inside the tile
        int ntile = 0;
        int c[kFillRowsPerWarp];
#pragma unroll
        for (int i = 0; i < kFillRowsPerWarp; ++i) {
            const int64_t s = __shfl_sync(kAll, rk, i);
            const int n = __shfl_sync(kAll, rem, i);
            c[i] = lane < n ? __ldg(indices + s + lane) : 0x7fffffff;
        }
#pragma unroll
        for (int i = 0; i < kFillRowsPerWarp; ++i) {
            int cc = c[i], taken = 0;
            for (int k = 0;;) {
                const bool in = cc < c_hi;
                const unsigned m = __ballot_sync(kAll, in);
                const int n_in = __popc(m);
                // sorted row: the tile's entries are a prefix of what follows the cursor, all >= c_lo
                bad |= (m != (n_in == 32 ? kAll : (1u << n_in) - 1u)) | (in && cc < c_lo);
                if (in && cc >= c_lo) atomicAdd(my_cur2 + ((cc - c_lo) >> 1), 1u << (16 * ((cc - c_lo) & 1)));
                taken += n_in;
                if (n_in < 32) break;
                // the row's segment is longer than the load issued up front
                k += 32;
                const int64_t s = __shfl_sync(kAll, rk, i);
                const int n = __shfl_sync(kAll, rem, i);
                cc = k + lane < n ? __ldg(indices + s + k + lane) : 0x7fffffff;
            }
            if (lane == i) ntile = taken;
        }
        __syncthreads();
        // thread j, column c_lo + j: exclusive scan over the warps, in warp (= row) order; the block's total must be
        // the count the write offsets were scanned from.  Then an exclusive scan of the totals over the tile's
        // columns places every column's run in the staging area.
        {
            const int j = threadIdx.x;
            uint32_t run = 0;
#pragma unroll
            for (int w = 0; w < kFillWarps; ++w) {
                const uint32_t cnt = wcur[w * kFillTileCols + j];
                wcur[w * kFillTileCols + j] = (uint16_t)run;
                run += cnt;
            }
            if (col_in) {
                bad |= run != want;
                cbase[j] = slot0;
            }
            uint32_t x = run;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t y = __shfl_up_sync(kAll, x, d);
                if (lane >= d) x += y;
            }
            if (lane == 31) wsum[warp] = x;
            __syncthreads();
            uint32_t off = 0;
            for (int w = 0; w < warp; ++w) off += wsum[w];
            cstart[j] = off + x - run;
            if (j == kFillTileCols - 1) cstart[kFillTileCols] = off + x;
        }
        __syncthreads();
        const bool staged = cstart[kFillTileCols] <= (uint32_t)kFillStage;          // CTA-uniform
        // walk 2: rows in order, each entry at the next slot of its (warp, column) cursor; the loads of a group of
        // rows are issued before the first of them is placed
        auto place = [&](int j, int r, float v) {
            const uint32_t o = my_cur[j]++;                // slot within the block's run of column c_lo + j
            if (staged) {
                const uint32_t p = cstart[j] + o;
                if (p < cstart[j + 1]) stage[p] = make_int2(r, __float_as_int(v));
            } else {
                const uint32_t slot = cbase[j] + o;
                if (slot < total) t_pairs[slot] = make_int2(r, __float_as_int(v));
            }
        };
        for (int g = 0; g < kFillRowsPerWarp; g += kFillGroup) {
            int c[kFillGroup];
            float v[kFillGroup];
#pragma unroll
            for (int i = 0; i < kFillGroup; ++i) {
                const int64_t s = __shfl_sync(kAll, rk, g + i);
                const int n = __shfl_sync(kAll, ntile, g + i);
                c[i] = lane < n ? ld_stream(indices + s + lane) : -1;
                v[i] = lane < n ? ld_stream(data + s + lane) : 0.f;
            }
#pragma unroll
            for (int i = 0; i < kFillGroup; ++i) {
                const int r = (int)(row0 + g + i);         // panel-local row index, as indptr starts at the panel
                if (c[i] >= c_lo && c[i] < c_hi) place(c[i] - c_lo, r, v[i]);
                const int n = __shfl_sync(kAll, ntile, g + i);
                if (n > 32) {
                    const int64_t s = __shfl_sync(kAll, rk, g + i);
                    for (int k = 32 + lane; k - lane < n; k += 32) {
                        const int cc = k < n ? ld_stream(indices + s + k) : -1;
                        const float vv = k < n ? ld_stream(data + s + k) : 0.f;
                        if (cc >= c_lo && cc < c_hi) place(cc - c_lo, r, vv);
                    }
                }
                __syncwarp();                              // row r's cursor updates land before row r + 1 reads them
            }
        }
        rk += ntile;
        rem -= ntile;
        __syncthreads();
        // every (block, column) run out of the staging area by consecutive lanes; cursors back to zero for the next tile
        if (staged) {
            for (int j = warp; j < c_hi - c_lo; j += kFillWarps) {
                const uint32_t p0 = cstart[j], n = cstart[j + 1] - p0, g0 = cbase[j];
                for (uint32_t e = lane; e < n; e += 32)
                    if (g0 + e < total) t_pairs[g0 + e] = stage[p0 + e];
            }
        }
        for (int j = threadIdx.x; j < kCurVecs; j += kFillThreads) reinterpret_cast<uint4*>(wcur)[j] = make_uint4(0u, 0u, 0u, 0u);
        __syncthreads();
    }
    if (t1 == n_tiles) bad |= rem != 0;                  // entries left over: a column >= n_cols (or unsorted)
    if (__syncthreads_or(bad) && threadIdx.x == 0) atomicOr(status, 1);
}

// per-row sum and sum of squares (fp64 accumulation); applied to the transposed panels of A this yields
// the per-feature moments MOFA's centring needs (intercepts, muon/_core/tools.py:283-286)
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

}  // namespace mub

extern "C" {

int mub_csr_transpose_fill_pairs(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_rows,
                                 int32_t n_cols, int64_t row_offset, const int64_t* t_indptr, int64_t* cursor,
                                 int32_t* t_pairs, mub_stream_t stream) {
    return mub::launch_transpose_fill<true, float>("transpose_fill_pairs", indptr, indices, data, n_rows, n_cols, row_offset,
                                            t_indptr, cursor, t_pairs, nullptr, stream);
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
    return mub::launch_transpose_fill<false>("transpose_fill", indptr, indices, data, n_rows, n_cols, row_offset,
                                             t_indptr, cursor, t_indices, t_data, stream);
}

int mub_csr_transpose_fill_f64(const int64_t* indptr, const int32_t* indices, const double* data, int64_t n_rows,
                               int32_t n_cols, int64_t row_offset, const int64_t* t_indptr, int64_t* cursor,
                               int32_t* t_indices, double* t_data, mub_stream_t stream) {
    return mub::launch_transpose_fill<false>("transpose_fill_f64", indptr, indices, data, n_rows, n_cols, row_offset,
                                             t_indptr, cursor, t_indices, t_data, stream);
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
    const size_t smem = mub::kFillSmem;
    cudaError_t e = cudaFuncSetAttribute(mub::transpose_fill_tiled_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess)      // room for two CTAs per SM
        e = cudaFuncSetAttribute(mub::transpose_fill_tiled_kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                                 (int)cudaSharedmemCarveoutMaxShared);
    if (e != cudaSuccess) {
        mub::set_error("transpose_fill_tiled: %zu B of shared memory: %s", smem, cudaGetErrorString(e));
        return -2;
    }
    // column slabs per row block: about 8 CTAs per SM in all, so that the last wave is short
    const int n_tiles = (int)((n_cols + mub::kFillTileCols - 1) / mub::kFillTileCols);
    int64_t slabs = (8ll * mub::sm_count() + n_blocks - 1) / n_blocks;
    slabs = slabs < 1 ? 1 : (slabs > n_tiles ? n_tiles : slabs);
    const int tiles_per_slab = (int)((n_tiles + slabs - 1) / slabs);
    const dim3 grid((unsigned)n_blocks, (unsigned)((n_tiles + tiles_per_slab - 1) / tiles_per_slab));
    mub::transpose_fill_tiled_kernel<<<grid, mub::kFillThreads, smem, s>>>(indptr, indices, data, n_rows, n_cols, tiles_per_slab,
                                                                          rb_count, base, t_indptr, (int2*)t_pairs, status);
    return mub::check_launch("transpose_fill_tiled");
}
