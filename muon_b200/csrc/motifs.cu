// Motif scanning (muon/_atac/tools.py:446-517, MOODS' forward-strand scan): score every window of every sequence
// against every log-odds matrix in float64, in column order from 0.0, and keep the windows scoring >= the motif's
// threshold.  A count pass and a fill pass run the same arithmetic; the fill pass writes each (sequence, motif, tile)
// run of hits at an offset from an exclusive scan of the counts, so the output is in (sequence, motif, position)
// order without float or order-dependent atomics, and two calls return identical bits.
#include "common.cuh"

namespace mub {

constexpr int kTile = MUB_MOTIF_TILE;              // window starts per CTA
constexpr int kThreads = 128;
constexpr int kPer = kTile / kThreads;             // consecutive window starts per thread
constexpr int kMaxLen = MUB_MOTIF_MAX_LEN;
constexpr int kCodes = MUB_MOTIF_CODES;            // A C G T, then "not a base" (score -inf)
constexpr int kGroupCols = MUB_MOTIF_GROUP_COLS;
static_assert(kTile % kThreads == 0, "tile must split evenly over the threads");

__global__ void motif_encode_kernel(uint8_t* __restrict__ b, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const unsigned c = b[i] | 0x20u;                 // ASCII lower case; non-letters never map to a-z below
        b[i] = c == 'a' ? 0 : c == 'c' ? 1 : c == 'g' ? 2 : c == 't' ? 3 : 4;
    }
}

struct ScanArgs {
    const uint8_t* codes;
    const int64_t* seq_off;      // [n_seq + 1] byte offsets of the sequences in codes
    const int32_t* tile_seq;     // [n_tiles] sequence of each tile
    const int64_t* seq_tile0;    // [n_seq + 1] first tile of each sequence
    const double* tab;           // [n_cols * kCodes]
    const int32_t* col_off;      // [n_motifs + 1]
    const double* thr;           // [n_motifs]
    const int32_t* group_m0;     // [n_groups + 1] first motif of each group
    int32_t n_groups, n_motifs;
    int32_t* counts;             // [n_tiles * n_motifs], laid out (sequence, motif, tile)
    const int64_t* offsets;      // exclusive scan of counts (fill pass only)
    int32_t* out_seq;
    int32_t* out_motif;
    int32_t* out_pos;
    double* out_score;
};

template <bool FILL>
__global__ void __launch_bounds__(kThreads) motif_scan_kernel(ScanArgs a) {
    extern __shared__ double tab_s[];                    // one group's columns, kCodes scores each
    __shared__ uint8_t seq_s[kTile + kMaxLen];
    __shared__ int cnt_s[kGroupCols];
    __shared__ int warp_s[2][kThreads / kWarp];
    const int64_t g = blockIdx.x;
    const int s = a.tile_seq[g];
    const int64_t t0 = a.seq_tile0[s], nt = a.seq_tile0[s + 1] - t0;
    const int64_t pos0 = (g - t0) * kTile;
    const int64_t base = a.seq_off[s], len = a.seq_off[s + 1] - base;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int w0 = threadIdx.x * kPer;
    for (int i = threadIdx.x; i < kTile + kMaxLen; i += kThreads) {
        const int64_t p = pos0 + i;                      // past the end reads as "not a base": no window runs over it
        seq_s[i] = p < len ? a.codes[base + p] : 4;
    }
    int parity = 0;
    for (int grp = blockIdx.y; grp < a.n_groups; grp += gridDim.y) {
        const int m0 = a.group_m0[grp], m1 = a.group_m0[grp + 1];
        const int c0 = a.col_off[m0], c1 = a.col_off[m1];
        __syncthreads();                                 // the previous group's table and counters are done with
        for (int i = threadIdx.x; i < (c1 - c0) * kCodes; i += kThreads) tab_s[i] = a.tab[(int64_t)c0 * kCodes + i];
        if (!FILL)
            for (int i = threadIdx.x; i < m1 - m0; i += kThreads) cnt_s[i] = 0;
        __syncthreads();
        for (int m = m0; m < m1; ++m) {
            const int64_t slot = t0 * a.n_motifs + (int64_t)m * nt + (g - t0);
            if (FILL && a.counts[slot] == 0) continue;   // uniform across the CTA
            const int L = a.col_off[m + 1] - a.col_off[m];
            const double* t = tab_s + (a.col_off[m] - c0) * kCodes;
            double sc[kPer];
            int c[kPer];
#pragma unroll
            for (int k = 0; k < kPer; ++k) {
                sc[k] = 0.0;
                c[k] = seq_s[w0 + k];
            }
            for (int j = 0; j < L; ++j) {                // c[k] is the base at w0 + k + j
                const double* col = t + j * kCodes;
#pragma unroll
                for (int k = 0; k < kPer; ++k) sc[k] += col[c[k]];
#pragma unroll
                for (int k = 0; k + 1 < kPer; ++k) c[k] = c[k + 1];
                c[kPer - 1] = seq_s[w0 + kPer + j];
            }
            const double th = a.thr[m];
            unsigned hit = 0;
#pragma unroll
            for (int k = 0; k < kPer; ++k) hit |= (sc[k] >= th ? 1u : 0u) << k;
            const int n = __popc(hit);
            if (!FILL) {
                const int wn = __reduce_add_sync(0xffffffffu, n);
                if (lane == 0 && wn) atomicAdd(&cnt_s[m - m0], wn);   // integer: the total is order-free
                continue;
            }
            int incl = n;                                // block exclusive scan of the per-thread hit counts
#pragma unroll
            for (int o = 1; o < kWarp; o <<= 1) {
                const int v = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += v;
            }
            if (lane == kWarp - 1) warp_s[parity][warp] = incl;
            __syncthreads();
            int before = 0;
            for (int w = 0; w < warp; ++w) before += warp_s[parity][w];
            parity ^= 1;                                 // the next scan's writes cannot race this one's reads
            int64_t o = a.offsets[slot] + before + incl - n;
#pragma unroll
            for (int k = 0; k < kPer; ++k)
                if (hit >> k & 1u) {
                    a.out_seq[o] = s;
                    a.out_motif[o] = m;
                    a.out_pos[o] = (int32_t)(pos0 + w0 + k);
                    a.out_score[o] = sc[k];
                    ++o;
                }
        }
        if (!FILL) {
            __syncthreads();
            for (int i = threadIdx.x; i < m1 - m0; i += kThreads)
                a.counts[t0 * a.n_motifs + (int64_t)(m0 + i) * nt + (g - t0)] = cnt_s[i];
        }
    }
}

template <bool FILL>
int launch_scan(const ScanArgs& a, int64_t n_tiles, cudaStream_t st) {
    MUB_REQUIRE(n_tiles >= 0 && n_tiles <= 0x7fffffff, "motif scan: %lld tiles", (long long)n_tiles);
    MUB_REQUIRE(a.n_groups >= 0 && a.n_motifs >= 0, "motif scan: negative motif or group count");
    if (n_tiles == 0 || a.n_groups == 0) return 0;
    const size_t smem = (size_t)kGroupCols * kCodes * sizeof(double);
    cudaFuncSetAttribute(motif_scan_kernel<FILL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    dim3 grid((unsigned)n_tiles, (unsigned)(a.n_groups < 65535 ? a.n_groups : 65535));
    motif_scan_kernel<FILL><<<grid, kThreads, smem, st>>>(a);
    return check_launch(FILL ? "motif_fill" : "motif_count");
}

}  // namespace mub

extern "C" {

int mub_motif_encode(uint8_t* bytes, int64_t n, mub_stream_t stream) {
    MUB_REQUIRE(n >= 0, "motif encode: n = %lld", (long long)n);
    if (n == 0) return 0;
    const int64_t blocks = (n + 255) / 256;
    const int grid = (int)(blocks < 8 * 1024 ? blocks : 8 * 1024);
    mub::motif_encode_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(bytes, n);
    return mub::check_launch("motif_encode");
}

int mub_motif_count(const uint8_t* codes, const int64_t* seq_off, const int32_t* tile_seq, const int64_t* seq_tile0,
                    int64_t n_tiles, const double* tab, const int32_t* col_off, const double* thr,
                    const int32_t* group_m0, int32_t n_groups, int32_t n_motifs, int32_t* counts,
                    mub_stream_t stream) {
    mub::ScanArgs a{codes, seq_off, tile_seq, seq_tile0, tab, col_off, thr, group_m0, n_groups, n_motifs, counts,
                    nullptr, nullptr, nullptr, nullptr, nullptr};
    return mub::launch_scan<false>(a, n_tiles, (cudaStream_t)stream);
}

int mub_motif_fill(const uint8_t* codes, const int64_t* seq_off, const int32_t* tile_seq, const int64_t* seq_tile0,
                   int64_t n_tiles, const double* tab, const int32_t* col_off, const double* thr,
                   const int32_t* group_m0, int32_t n_groups, int32_t n_motifs, const int32_t* counts,
                   const int64_t* offsets, int32_t* out_seq, int32_t* out_motif, int32_t* out_pos, double* out_score,
                   mub_stream_t stream) {
    mub::ScanArgs a{codes, seq_off, tile_seq, seq_tile0, tab, col_off, thr, group_m0, n_groups, n_motifs,
                    const_cast<int32_t*>(counts), offsets, out_seq, out_motif, out_pos, out_score};
    return mub::launch_scan<true>(a, n_tiles, (cudaStream_t)stream);
}

}  // extern "C"
