// Fragments file (muon/_atac/tools.py:746-1201): split and parse inflated text chunks, look barcodes up in an
// open-addressing table, then count fragments over feature windows, pile them up around TSSs, or classify their
// lengths.  Every count is an integer atomic, so results are exact and two calls return identical bits.
#include "common.cuh"

namespace mub {

constexpr int kNlThreads = 256;
constexpr int kNlIters = 16;
constexpr int64_t kNlTile = (int64_t)kNlThreads * kNlIters;   // bytes per tile of the newline scan

// ---- line split: newline positions in byte order (ballot per warp, scan across warps, tiles in order) ----------------
__global__ void newline_count_kernel(const uint8_t* __restrict__ text, int64_t n, int64_t* __restrict__ tile_counts) {
    __shared__ int warp_n[kNlThreads / kWarp];
    const int64_t base = (int64_t)blockIdx.x * kNlTile;
    int c = 0;
    for (int j = 0; j < kNlIters; ++j) {
        const int64_t i = base + (int64_t)j * kNlThreads + threadIdx.x;
        c += (i < n && text[i] == '\n');
    }
    for (int o = 16; o; o >>= 1) c += __shfl_down_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0) warp_n[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        int64_t t = 0;
        for (int w = 0; w < kNlThreads / kWarp; ++w) t += warp_n[w];
        tile_counts[blockIdx.x] = t;
    }
}

__global__ void newline_fill_kernel(const uint8_t* __restrict__ text, int64_t n, const int64_t* __restrict__ tile_off,
                                    int64_t* __restrict__ nl_pos) {
    __shared__ int warp_n[kNlThreads / kWarp];
    const int64_t base = (int64_t)blockIdx.x * kNlTile;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int64_t run = tile_off[blockIdx.x];
    for (int j = 0; j < kNlIters; ++j) {
        const int64_t i = base + (int64_t)j * kNlThreads + threadIdx.x;
        const bool nl = i < n && text[i] == '\n';
        const unsigned b = __ballot_sync(0xffffffffu, nl);
        if (lane == 0) warp_n[warp] = __popc(b);
        __syncthreads();
        int before = 0, total = 0;
        for (int w = 0; w < kNlThreads / kWarp; ++w) {
            before += w < warp ? warp_n[w] : 0;
            total += warp_n[w];
        }
        if (nl) nl_pos[run + before + __popc(b & ((1u << lane) - 1u))] = i;
        run += total;
        __syncthreads();
    }
}

// ---- barcode table ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t bc_hash(const uint8_t* p, int64_t len) {
    uint64_t h = 1469598103934665603ull;                 // FNV-1a, then a murmur finaliser
    for (int64_t k = 0; k < len; ++k) h = (h ^ p[k]) * 1099511628211ull;
    h ^= h >> 33;
    h *= 0xff51afd7ed558ccdull;
    h ^= h >> 33;
    return h ? h : 1;                                     // 0 marks an empty slot
}

__global__ void barcode_insert_kernel(const uint8_t* __restrict__ bc, const int64_t* __restrict__ bc_off, int32_t n_bc,
                                      unsigned long long* keys, int32_t* __restrict__ slot_entry, int64_t mask) {
    const int32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_bc) return;
    const unsigned long long h = bc_hash(bc + bc_off[j], bc_off[j + 1] - bc_off[j]);
    for (int64_t s = (int64_t)(h & mask);; s = (s + 1) & mask) {
        if (atomicCAS(&keys[s], 0ull, h) == 0ull) {
            slot_entry[s] = j;
            return;
        }
    }
}

// ---- parse: one thread per line ---------------------------------------------------------------------------------------
struct ParseStatus {           // int64 words, initialised by the caller to {MAX, MAX, MAX, 0, 0}
    enum { kMalformed = 0, kOverflow = 1, kUnsorted = 2, kLmax = 3, kSkipped = 4 };
};

__device__ __forceinline__ bool parse_uint(const uint8_t* p, int64_t a, int64_t b, int64_t& v) {
    if (a >= b) return false;
    int64_t x = 0;
    for (int64_t k = a; k < b; ++k) {
        const unsigned d = p[k] - '0';
        if (d > 9) return false;
        x = x * 10 + d;
        if (x > (int64_t)1 << 40) x = (int64_t)1 << 40;  // saturate: flagged as overflow below
    }
    v = x;
    return true;
}

__global__ void parse_kernel(const uint8_t* __restrict__ text, const int64_t* __restrict__ nl, int64_t n_lines,
                             int64_t line_base, const uint8_t* __restrict__ bc, const int64_t* __restrict__ bc_off,
                             const int32_t* __restrict__ bc_val, const unsigned long long* __restrict__ keys,
                             const int32_t* __restrict__ slot_entry, int64_t mask, int32_t* __restrict__ start,
                             int32_t* __restrict__ end, int32_t* __restrict__ score, int32_t* __restrict__ cell,
                             uint8_t* __restrict__ flags, unsigned long long* status) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_lines) return;
    const int64_t a = i ? nl[i - 1] + 1 : 0, b = nl[i];
    start[i] = 0;
    end[i] = 0;
    score[i] = 0;
    cell[i] = -1;
    if (b > a && text[a] == '#') {
        flags[i] = 2;
        atomicAdd(&status[ParseStatus::kSkipped], 1ull);
        return;
    }
    int64_t tab[4];
    int nt = 0;
    for (int64_t k = a; k < b && nt < 4; ++k)
        if (text[k] == '\t') tab[nt++] = k;
    int64_t f5 = b;                                       // the score ends at the 5th tab or at the end of the line
    if (nt == 4)
        for (int64_t k = tab[3] + 1; k < b; ++k)
            if (text[k] == '\t') {
                f5 = k;
                break;
            }
    int64_t s = 0, e = 0, sc = 0;
    bool ok = nt == 4 && tab[0] > a && parse_uint(text, tab[0] + 1, tab[1], s) && parse_uint(text, tab[1] + 1, tab[2], e);
    if (ok) {
        const bool neg = tab[3] + 1 < f5 && text[tab[3] + 1] == '-';
        ok = parse_uint(text, tab[3] + 1 + neg, f5, sc);
        if (neg) sc = -sc;
    }
    if (!ok) {
        atomicMin(&status[ParseStatus::kMalformed], (unsigned long long)(line_base + i));
        flags[i] = 0;
        return;
    }
    if (s > 2147483647 || e > 2147483647 || sc > 2147483647 || sc < -2147483647)
        atomicMin(&status[ParseStatus::kOverflow], (unsigned long long)(line_base + i));
    start[i] = (int32_t)min(s, (int64_t)2147483647);
    end[i] = (int32_t)min(e, (int64_t)2147483647);
    score[i] = (int32_t)max(min(sc, (int64_t)2147483647), (int64_t)-2147483647);
    if (e > s) atomicMax(&status[ParseStatus::kLmax], (unsigned long long)(e - s));

    // run start: first line of the chunk, or a chromosome that differs from the previous line's
    bool run = true;
    if (i > 0) {
        const int64_t pa = i > 1 ? nl[i - 2] + 1 : 0, pb = nl[i - 1];
        const int64_t len = tab[0] - a;
        if (pb - pa > len && text[pa + len] == '\t') {
            run = false;
            for (int64_t k = 0; k < len; ++k)
                if (text[pa + k] != text[a + k]) {
                    run = true;
                    break;
                }
            if (!run) {          // same chromosome: starts never decrease
                int64_t ps = 0;
                int64_t q = pa + len + 1, qe = q;
                while (qe < pb && text[qe] != '\t') ++qe;
                if (parse_uint(text, q, qe, ps) && s < ps)
                    atomicMin(&status[ParseStatus::kUnsorted], (unsigned long long)(line_base + i));
            }
        }
    }
    flags[i] = run ? 1 : 0;

    // barcode -> obs index: hash probe, every hit confirmed by a byte compare
    const uint8_t* name = text + tab[2] + 1;
    const int64_t nlen = tab[3] - tab[2] - 1;
    const unsigned long long h = bc_hash(name, nlen);
    if (keys == nullptr) return;
    for (int64_t q = (int64_t)(h & mask);; q = (q + 1) & mask) {
        const unsigned long long k = keys[q];
        if (k == 0ull) break;
        if (k != h) continue;
        const int32_t j = slot_entry[q];
        const int64_t o = bc_off[j];
        if (bc_off[j + 1] - o != nlen) continue;
        bool eq = true;
        for (int64_t t = 0; t < nlen; ++t)
            if (bc[o + t] != name[t]) {
                eq = false;
                break;
            }
        if (eq) {
            cell[i] = bc_val[j];
            break;
        }
    }
}

// ---- interval overlap: one warp per query over its contig's start-sorted records --------------------------------------
// records [rec_lo, rec_hi) of the query's contig; the first candidate is the first start >= lo - lmax + 1
__device__ __forceinline__ int64_t first_candidate(const int32_t* __restrict__ start, int64_t l, int64_t h, int64_t key) {
    while (l < h) {
        const int64_t m = (l + h) >> 1;
        if ((int64_t)start[m] < key) l = m + 1;
        else h = m;
    }
    return l;
}

template <int MODE>   // 0: count hits, 1: emit (cell, feature, value), 2: TSS difference array
__global__ void overlap_kernel(const int32_t* __restrict__ start, const int32_t* __restrict__ end,
                               const int32_t* __restrict__ cell, const int32_t* __restrict__ score,
                               const int64_t* __restrict__ q_rec_lo, const int64_t* __restrict__ q_rec_hi,
                               const int64_t* __restrict__ q_lo, const int64_t* __restrict__ q_hi, int32_t n_q,
                               int64_t lmax, int32_t use_score, int32_t feat_base, int64_t* __restrict__ counts,
                               const int64_t* __restrict__ out_off, int32_t* __restrict__ out_cell,
                               int32_t* __restrict__ out_feat, int64_t* __restrict__ out_val, int32_t width,
                               unsigned long long* __restrict__ diff) {
    const int64_t gw = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (gw >= n_q) return;
    const int64_t lo = q_lo[gw], hi = q_hi[gw], rh = q_rec_hi[gw];
    int64_t j = first_candidate(start, q_rec_lo[gw], rh, lo - lmax + 1);
    int64_t n_hit = 0, w = MODE == 1 ? out_off[gw] : 0;
    for (; j < rh; j += 32) {
        const int64_t r = j + lane;
        const bool in = r < rh && (int64_t)start[r] < hi;
        const int32_t c = in ? cell[r] : -1;
        const bool hit = in && (int64_t)end[r] > lo && c >= 0;
        const unsigned bh = __ballot_sync(0xffffffffu, hit);
        if (MODE == 1 && hit) {
            const int64_t o = w + __popc(bh & ((1u << lane) - 1u));
            out_cell[o] = c;
            out_feat[o] = feat_base + (int32_t)gw;
            out_val[o] = use_score ? (int64_t)score[r] : 1;
        }
        if (MODE == 2 && hit) {
            const int64_t cs = max((int64_t)start[r] - lo, (int64_t)0);
            const int64_t ce = min((int64_t)end[r] - lo, (int64_t)width);
            if (ce > cs) {
                unsigned long long* row = diff + (int64_t)c * (width + 1);
                const long long v = score[r];
                atomicAdd(row + cs, (unsigned long long)v);
                atomicAdd(row + ce, (unsigned long long)(-v));
            }
        }
        w += __popc(bh);
        n_hit += __popc(bh);
        if (__ballot_sync(0xffffffffu, r < rh && !in)) break;   // passed hi: the rest start later
    }
    if (MODE == 0 && lane == 0) counts[gw] = n_hit;
}

// ---- TSS rows: one warp per cell turns its difference row into the pileup and the exact flank / centre sums ----------
__global__ void tss_rows_kernel(long long* __restrict__ diff, int64_t n_cells, int32_t width, int32_t flank,
                                int32_t c_lo, int32_t c_hi, long long* __restrict__ sums) {
    const int64_t c = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (c >= n_cells) return;
    long long* row = diff + c * (int64_t)(width + 1);
    long long carry = 0, fl = 0, ce = 0;
    for (int32_t base = 0; base < width; base += 32) {
        const int32_t p = base + lane;
        long long v = p < width ? row[p] : 0;
        for (int o = 1; o < 32; o <<= 1) {
            const long long u = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= o) v += u;
        }
        v += carry;
        carry = __shfl_sync(0xffffffffu, v, 31);
        if (p < width) {
            row[p] = v;
            if (p < flank || p >= width - flank) fl += v;
            if (p >= c_lo && p < c_hi) ce += v;
        }
    }
    for (int o = 16; o; o >>= 1) {
        fl += __shfl_down_sync(0xffffffffu, fl, o);
        ce += __shfl_down_sync(0xffffffffu, ce, o);
    }
    if (lane == 0) {
        sums[2 * c] = fl;
        sums[2 * c + 1] = ce;
    }
}

__global__ void tss_scale_kernel(const long long* __restrict__ pile, int64_t n_cells, int32_t width,
                                 const double* __restrict__ flank_mean, double* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_cells * width) return;
    const int64_t c = i / width, p = i - c * width;
    out[i] = (double)pile[c * (width + 1) + p] / flank_mean[c];
}

// ---- nucleosome classes over the first n records ---------------------------------------------------------------------
__global__ void nucleosome_kernel(const int32_t* __restrict__ start, const int32_t* __restrict__ end,
                                  const int32_t* __restrict__ cell, int64_t n, double free_ub, double mono_ub,
                                  int32_t* __restrict__ counts) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t c = cell[i];
    if (c < 0) return;
    const double len = (double)((int64_t)end[i] - (int64_t)start[i]);
    if (len < free_ub) atomicAdd(counts + 2 * (int64_t)c, 1);
    else if (len < mono_ub) atomicAdd(counts + 2 * (int64_t)c + 1, 1);
}

inline unsigned blocks_for(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }

}  // namespace mub

extern "C" {

int64_t mub_frag_tile_bytes(void) { return mub::kNlTile; }

int mub_frag_newline_count(const uint8_t* text, int64_t n_bytes, int64_t* tile_counts, mub_stream_t stream) {
    MUB_REQUIRE(n_bytes >= 0, "frag_newline_count: bad size");
    if (n_bytes == 0) return 0;
    MUB_REQUIRE(text && tile_counts, "frag_newline_count: null pointer");
    const int64_t tiles = (n_bytes + mub::kNlTile - 1) / mub::kNlTile;
    MUB_REQUIRE(tiles < (1ll << 31), "frag_newline_count: chunk too large");
    mub::newline_count_kernel<<<(unsigned)tiles, mub::kNlThreads, 0, (cudaStream_t)stream>>>(text, n_bytes, tile_counts);
    return mub::check_launch("frag_newline_count");
}

int mub_frag_newline_fill(const uint8_t* text, int64_t n_bytes, const int64_t* tile_offsets, int64_t* nl_pos,
                          mub_stream_t stream) {
    MUB_REQUIRE(n_bytes >= 0, "frag_newline_fill: bad size");
    if (n_bytes == 0) return 0;
    MUB_REQUIRE(text && tile_offsets && nl_pos, "frag_newline_fill: null pointer");
    const int64_t tiles = (n_bytes + mub::kNlTile - 1) / mub::kNlTile;
    MUB_REQUIRE(tiles < (1ll << 31), "frag_newline_fill: chunk too large");
    mub::newline_fill_kernel<<<(unsigned)tiles, mub::kNlThreads, 0, (cudaStream_t)stream>>>(text, n_bytes, tile_offsets,
                                                                                            nl_pos);
    return mub::check_launch("frag_newline_fill");
}

int mub_frag_barcode_table(const uint8_t* bc, const int64_t* bc_off, int32_t n_bc, uint64_t* keys, int32_t* slot_entry,
                           int64_t capacity, mub_stream_t stream) {
    MUB_REQUIRE(n_bc >= 0 && capacity > n_bc && (capacity & (capacity - 1)) == 0,
                "frag_barcode_table: capacity %lld must be a power of two above %d", (long long)capacity, n_bc);
    if (n_bc == 0) return 0;
    MUB_REQUIRE(bc && bc_off && keys && slot_entry, "frag_barcode_table: null pointer");
    mub::barcode_insert_kernel<<<mub::blocks_for(n_bc, 256), 256, 0, (cudaStream_t)stream>>>(
        bc, bc_off, n_bc, (unsigned long long*)keys, slot_entry, capacity - 1);
    return mub::check_launch("frag_barcode_table");
}

int mub_frag_parse(const uint8_t* text, const int64_t* nl_pos, int64_t n_lines, int64_t line_base, const uint8_t* bc,
                   const int64_t* bc_off, const int32_t* bc_val, const uint64_t* keys, const int32_t* slot_entry,
                   int64_t capacity, int32_t* start, int32_t* end, int32_t* score, int32_t* cell, uint8_t* flags,
                   int64_t* status, mub_stream_t stream) {
    MUB_REQUIRE(n_lines >= 0, "frag_parse: bad size");
    if (n_lines == 0) return 0;
    MUB_REQUIRE(text && nl_pos && start && end && score && cell && flags && status, "frag_parse: null pointer");
    MUB_REQUIRE(keys == nullptr || (capacity > 0 && (capacity & (capacity - 1)) == 0 && bc_off && bc_val && slot_entry),
                "frag_parse: bad barcode table");
    mub::parse_kernel<<<mub::blocks_for(n_lines, 256), 256, 0, (cudaStream_t)stream>>>(
        text, nl_pos, n_lines, line_base, bc, bc_off, bc_val, (const unsigned long long*)keys, slot_entry, capacity - 1,
        start, end, score, cell, flags, (unsigned long long*)status);
    return mub::check_launch("frag_parse");
}

int mub_frag_overlap(const int32_t* start, const int32_t* end, const int32_t* cell, const int32_t* score,
                     const int64_t* q_rec_lo, const int64_t* q_rec_hi, const int64_t* q_lo, const int64_t* q_hi,
                     int32_t n_q, int64_t lmax, int32_t use_score, int32_t feat_base, int64_t* counts,
                     const int64_t* out_off, int32_t* out_cell, int32_t* out_feat, int64_t* out_val,
                     mub_stream_t stream) {
    MUB_REQUIRE(n_q >= 0 && lmax >= 0, "frag_overlap: bad shape");
    if (n_q == 0) return 0;
    MUB_REQUIRE(start && end && cell && q_rec_lo && q_rec_hi && q_lo && q_hi, "frag_overlap: null pointer");
    const unsigned grid = mub::blocks_for((int64_t)n_q * 32, 256);
    if (out_off == nullptr) {
        MUB_REQUIRE(counts, "frag_overlap: null counts");
        mub::overlap_kernel<0><<<grid, 256, 0, (cudaStream_t)stream>>>(start, end, cell, score, q_rec_lo, q_rec_hi, q_lo,
                                                                       q_hi, n_q, lmax, use_score, feat_base, counts,
                                                                       nullptr, nullptr, nullptr, nullptr, 0, nullptr);
    } else {
        MUB_REQUIRE(out_cell && out_feat && out_val && (score || !use_score), "frag_overlap: null output");
        mub::overlap_kernel<1><<<grid, 256, 0, (cudaStream_t)stream>>>(start, end, cell, score, q_rec_lo, q_rec_hi, q_lo,
                                                                       q_hi, n_q, lmax, use_score, feat_base, nullptr,
                                                                       out_off, out_cell, out_feat, out_val, 0, nullptr);
    }
    return mub::check_launch("frag_overlap");
}

int mub_frag_tss_pileup(const int32_t* start, const int32_t* end, const int32_t* cell, const int32_t* score,
                        const int64_t* q_rec_lo, const int64_t* q_rec_hi, const int64_t* q_lo, const int64_t* q_hi,
                        int32_t n_q, int64_t lmax, int32_t width, int64_t* diff, mub_stream_t stream) {
    MUB_REQUIRE(n_q >= 0 && lmax >= 0 && width > 0, "frag_tss_pileup: bad shape");
    if (n_q == 0) return 0;
    MUB_REQUIRE(start && end && cell && score && q_rec_lo && q_rec_hi && q_lo && q_hi && diff,
                "frag_tss_pileup: null pointer");
    mub::overlap_kernel<2><<<mub::blocks_for((int64_t)n_q * 32, 256), 256, 0, (cudaStream_t)stream>>>(
        start, end, cell, score, q_rec_lo, q_rec_hi, q_lo, q_hi, n_q, lmax, 1, 0, nullptr, nullptr, nullptr, nullptr,
        nullptr, width, (unsigned long long*)diff);
    return mub::check_launch("frag_tss_pileup");
}

int mub_frag_tss_rows(int64_t* diff, int64_t n_cells, int32_t width, int32_t flank, int32_t center_lo,
                      int32_t center_hi, int64_t* sums, mub_stream_t stream) {
    MUB_REQUIRE(n_cells >= 0 && width > 0 && flank >= 0 && center_lo <= center_hi, "frag_tss_rows: bad shape");
    if (n_cells == 0) return 0;
    MUB_REQUIRE(diff && sums, "frag_tss_rows: null pointer");
    mub::tss_rows_kernel<<<mub::blocks_for(n_cells * 32, 256), 256, 0, (cudaStream_t)stream>>>(
        (long long*)diff, n_cells, width, flank, center_lo, center_hi, (long long*)sums);
    return mub::check_launch("frag_tss_rows");
}

int mub_frag_tss_scale(const int64_t* pile, int64_t n_cells, int32_t width, const double* flank_mean, double* out,
                       mub_stream_t stream) {
    MUB_REQUIRE(n_cells >= 0 && width > 0, "frag_tss_scale: bad shape");
    if (n_cells == 0) return 0;
    MUB_REQUIRE(pile && flank_mean && out, "frag_tss_scale: null pointer");
    mub::tss_scale_kernel<<<mub::blocks_for(n_cells * width, 256), 256, 0, (cudaStream_t)stream>>>(
        (const long long*)pile, n_cells, width, flank_mean, out);
    return mub::check_launch("frag_tss_scale");
}

int mub_frag_nucleosome(const int32_t* start, const int32_t* end, const int32_t* cell, int64_t n, double free_ub,
                        double mono_ub, int32_t* counts, mub_stream_t stream) {
    MUB_REQUIRE(n >= 0, "frag_nucleosome: bad size");
    if (n == 0) return 0;
    MUB_REQUIRE(start && end && cell && counts, "frag_nucleosome: null pointer");
    mub::nucleosome_kernel<<<mub::blocks_for(n, 256), 256, 0, (cudaStream_t)stream>>>(start, end, cell, n, free_ub,
                                                                                      mono_ub, counts);
    return mub::check_launch("frag_nucleosome");
}

}  // extern "C"
