// Leiden / Louvain community detection: the device steps of one level (reference muon/_core/tools.py:928-1206,
// which hands the multiplex RB-configuration problem to leidenalg / louvain-igraph).
//
// The host (_leiden.py) collapses the multiplex objective  sum_l w_l sum_ij (A^l_ij - g_l k^l_i k^l_j / m_l) d(s_i, s_j)
// to one graph (weights sum_l w_l A^l_uv) plus per-layer degrees k^l_v and constants c_l = w_l g_l / m_l, so the
// kernels never see layers.  Weights and degrees arrive as int64 fixed point (scales 2^Se, 2^Sk chosen by the host so
// every total stays below 2^53): every sum over entries or vertices is an exact integer sum, so atomics cannot change
// a result and every launch is bit-identical from run to run.
//
//   scan   : one warp per vertex v.  The warp gathers e_{v,c} = sum of w_vu over the neighbours u != v in community c
//            into a per-warp open-addressing table (shared memory; rows longer than kMaxDeg use a table sized from
//            their degree in global memory, a second launch), then scores every candidate
//                s(c) = e_{v,c} ce - sum_l c'_l k^l_v K^l_c
//            in fp64 with a fixed operation order (no contraction) and keeps the best, ties to the smaller id.
//            mode 0 (local moving): candidates are the neighbour communities and an empty one (id n + v); the gain
//            2 (s(b) - s(own)) is evaluated from exact integer differences and proposed only above a relative
//            rounding margin.  mode 1 (refinement): only singletons of the refined partition move, to sub-communities
//            of the same parent that they touch, with a non-negative gain; a hashed coin per (round, vertex) splits
//            the singletons into movers and frozen ones, and no mover may target a moving singleton.
//   apply  : mode 0 (local moving): every proposal carries a unique hashed priority (written to prio); the proposals
//            whose priority is >= min_priority move.  The host then checks the sweep's exact change of quality from
//            the fixed-point totals and, if it is not positive, repeats the apply with the higher-priority half of
//            those movers (no rescan): every accepted sweep strictly raises the quality, so local moving terminates
//            without an iteration cap, while many vertices may join one community in the same sweep.
//            mode 1 (refinement): every proposal moves.
//   totals : per-community degree totals K^l_c and sizes (exact integer atomics).
//   segment_sum / internal : the aggregate graph's reduce and the internal weight of a partition.
#include <math.h>

#include "common.cuh"

namespace mub {
namespace leiden {

constexpr int kWarps = 4;
constexpr int kSlots = 512;             // hash slots per warp in shared memory
constexpr int kMaxDeg = kSlots / 2;     // longer rows go to the global-memory (hub) launch
constexpr int kThreads = 256;

struct Table {
    int32_t* key;                   // [H] -1 = empty
    unsigned long long* val;        // [H] fixed-point weight sums
    int32_t* list;                  // occupied slots (<= row length)
    int* count;
    int H;
    int shift;
};

__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

// per-vertex hash of a stream key: priorities (local moving) and coins (refinement)
__device__ __forceinline__ uint64_t vertex_hash(uint64_t key, int64_t v) {
    return splitmix64(key ^ ((uint64_t)v * 0xD1B54A32D192ED03ull));
}
__device__ __forceinline__ unsigned long long priority(uint64_t key, int64_t v) {
    return (1ull << 63) | ((vertex_hash(key, v) >> 33) << 32) | (uint64_t)(uint32_t)v;
}
__device__ __forceinline__ bool coin(uint64_t key, int64_t v) { return (vertex_hash(key, v) >> 63) != 0; }

__device__ __forceinline__ void table_add(const Table& t, int32_t c, long long w) {
    uint32_t h = ((uint32_t)c * 2654435761u) >> t.shift;
    while (true) {
        const int32_t old = atomicCAS(&t.key[h], -1, c);
        if (old == -1) {
            t.list[atomicAdd(t.count, 1)] = (int32_t)h;
            atomicAdd(&t.val[h], (unsigned long long)w);
            return;
        }
        if (old == c) {
            atomicAdd(&t.val[h], (unsigned long long)w);
            return;
        }
        h = (h + 1) & (t.H - 1);     // H >= 2 x row length: never full
    }
}

struct Problem {
    const int64_t* indptr;
    const int32_t* indices;
    const int64_t* w;        // [nnz] fixed-point combined weights
    const int64_t* k;        // [n x L] fixed-point degrees
    int64_t n;
    int L;
    double ce;               // 2^-Se
    double cl[4];            // c_l 2^-2Sk
};

struct State {
    const int32_t* memb;     // mode 0: communities; mode 1: refined sub-communities
    const int32_t* parent;   // mode 1: communities (the refinement stays inside them)
    const int64_t* K;        // [cap x L] totals of memb
    const int32_t* size;     // [cap]
    uint64_t key;
    int32_t* target;         // [n] -1 = stay
    double* gain;            // [n]
    int32_t* flags;          // bit 0: a singleton still has a non-negative move (mode 1)
};

constexpr double kMargin = 9.094947017729282e-13;   // 2^-40: moves whose gain is within rounding of 0 are not taken

// s(c) = e ce - sum_l (c'_l k_l) K_l, in this order, without contraction (the numpy restatement computes the same)
__device__ __forceinline__ double score(const Problem& P, long long e, const int64_t* kv, const int64_t* Kc) {
    double acc = 0.0;
    for (int l = 0; l < P.L; ++l) acc = __dadd_rn(acc, __dmul_rn(__dmul_rn(P.cl[l], (double)kv[l]), (double)Kc[l]));
    return __dadd_rn(__dmul_rn((double)e, P.ce), -acc);
}

template <int MODE>
__device__ void scan_vertex(const Problem& P, const State& S, const Table& T, int64_t v, int lane) {
    const int64_t p0 = P.indptr[v], p1 = P.indptr[v + 1];
    const int32_t own = S.memb[v];
    const int32_t pv = MODE == 1 ? S.parent[v] : 0;
    const int64_t* kv = P.k + v * P.L;
    if (MODE == 1 && S.size[own] != 1) {        // only singletons move in the refinement
        if (lane == 0) {
            S.target[v] = -1;
            S.gain[v] = 0.0;
        }
        return;
    }
    for (int64_t e = p0 + lane; e < p1; e += 32) {
        const int32_t u = P.indices[e];
        if (u == (int32_t)v) continue;
        if (MODE == 1 && S.parent[u] != pv) continue;
        table_add(T, S.memb[u], (long long)P.w[e]);
    }
    __syncwarp();
    const int nd = *T.count;
    const bool mover = MODE == 0 || coin(S.key, v);
    double best = -INFINITY;
    int32_t best_c = 0x7fffffff;
    long long e_best = 0, e_own = 0;
    bool any = false;
    for (int i = lane; i < nd; i += 32) {
        const int h = T.list[i];
        const int32_t c = T.key[h];
        const long long ev = (long long)T.val[h];
        if (MODE == 0 && c == own) {
            e_own = ev;
            continue;
        }
        const double s = score(P, ev, kv, S.K + (int64_t)c * P.L);
        if (MODE == 1) {
            any |= s >= 0.0;
            if (S.size[c] == 1 && coin(S.key, c)) continue;   // a moving singleton is not a target this round
        }
        if (s > best || (s == best && c < best_c)) {
            best = s;
            best_c = c;
            e_best = ev;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int32_t oc = __shfl_xor_sync(0xffffffffu, best_c, o);
        const long long oe = __shfl_xor_sync(0xffffffffu, e_best, o);
        if (ob > best || (ob == best && oc < best_c)) {
            best = ob;
            best_c = oc;
            e_best = oe;
        }
        e_own += __shfl_xor_sync(0xffffffffu, e_own, o);
    }
    any = __any_sync(0xffffffffu, any);
    // reset the touched slots for the next row
    __syncwarp();
    for (int i = lane; i < nd; i += 32) {
        const int h = T.list[i];
        T.key[h] = -1;
        T.val[h] = 0ull;
    }
    __syncwarp();
    if (lane != 0) return;
    *T.count = 0;
    if (MODE == 1) {
        const bool take = mover && best_c != 0x7fffffff && best >= 0.0;
        S.target[v] = take ? best_c : -1;
        S.gain[v] = take ? 2.0 * best : 0.0;
        if (any && !take) atomicOr(S.flags, 1);
        return;
    }
    // local moving: the best existing candidate, or an empty community when v is not alone (ties: existing)
    const int64_t* Ka = S.K + (int64_t)own * P.L;
    const bool empty_ok = S.size[own] > 1;
    const bool has_c = best_c != 0x7fffffff;
    const bool to_empty = empty_ok && (!has_c || best < 0.0);
    int32_t b = -1;
    double g = 0.0;
    if (has_c || to_empty) {
        const long long de = (to_empty ? 0ll : e_best) - e_own;
        const int64_t* Kb = to_empty ? nullptr : S.K + (int64_t)best_c * P.L;
        double acc = 0.0, mag = 0.0;
        for (int l = 0; l < P.L; ++l) {
            const long long dK = (Kb ? Kb[l] : 0ll) - Ka[l] + kv[l];
            const double t = __dmul_rn(__dmul_rn(P.cl[l], (double)kv[l]), (double)dK);
            acc = __dadd_rn(acc, t);
            mag = __dadd_rn(mag, fabs(t));
        }
        const double ex = __dmul_rn((double)de, P.ce);
        g = 2.0 * __dadd_rn(ex, -acc);
        const double scale = 2.0 * __dadd_rn(fabs(ex), mag);
        if (g > kMargin * scale) b = to_empty ? (int32_t)(P.n + v) : best_c;
    }
    S.target[v] = b;
    S.gain[v] = b >= 0 ? g : 0.0;
}

__device__ __forceinline__ Table carve_shared(unsigned char* base, int warp, int* counts) {
    Table t;
    unsigned char* p = base + (size_t)warp * (kSlots * (sizeof(int32_t) + sizeof(unsigned long long)) +
                                              kMaxDeg * sizeof(int32_t));
    t.val = reinterpret_cast<unsigned long long*>(p);
    t.key = reinterpret_cast<int32_t*>(t.val + kSlots);
    t.list = t.key + kSlots;
    t.count = counts + warp;
    t.H = kSlots;
    t.shift = 32 - 9;
    return t;
}
constexpr size_t kSmemPerWarp = kSlots * (sizeof(int32_t) + sizeof(unsigned long long)) + kMaxDeg * sizeof(int32_t);

template <int MODE>
__global__ void __launch_bounds__(kWarps * 32) scan_kernel(Problem P, State S) {
    __shared__ __align__(16) unsigned char smem[kSmemPerWarp * kWarps];
    __shared__ int counts[kWarps];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const Table T = carve_shared(smem, warp, counts);
    for (int h = lane; h < kSlots; h += 32) {
        T.key[h] = -1;
        T.val[h] = 0ull;
    }
    if (lane == 0) *T.count = 0;
    __syncwarp();
    for (int64_t v = (int64_t)blockIdx.x * kWarps + warp; v < P.n; v += (int64_t)gridDim.x * kWarps) {
        if (P.indptr[v + 1] - P.indptr[v] > kMaxDeg) continue;      // the hub launch takes it
        scan_vertex<MODE>(P, S, T, v, lane);
        __syncwarp();
    }
}

// hub rows: one warp per row, table of hub_H[i] (a power of two >= 2 x degree) slots at hub_off[i]
template <int MODE>
__global__ void __launch_bounds__(kWarps * 32)
scan_hub_kernel(Problem P, State S, const int32_t* __restrict__ hubs, int64_t n_hubs, const int64_t* __restrict__ off,
                const int32_t* __restrict__ Hs, int32_t* keys, unsigned long long* vals, int32_t* lists,
                int32_t* cnts) {
    const int lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (i >= n_hubs) return;
    Table T;
    T.H = Hs[i];
    T.shift = 32 - (31 - __clz(T.H));
    T.key = keys + off[i];
    T.val = vals + off[i];
    T.list = lists + off[i] / 2;
    T.count = cnts + i;
    for (int h = lane; h < T.H; h += 32) {
        T.key[h] = -1;
        T.val[h] = 0ull;
    }
    if (lane == 0) *T.count = 0;
    __syncwarp();
    scan_vertex<MODE>(P, S, T, hubs[i], lane);
}

__global__ void apply_kernel(int mode, int64_t n, int32_t* memb, const int32_t* __restrict__ target, uint64_t key,
                             unsigned long long min_priority, unsigned long long* prio, int32_t* counts) {
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= n) return;
    const int32_t b = target[v];
    if (mode == 0) {
        const unsigned long long p = b >= 0 ? priority(key, v) : 0ull;
        prio[v] = p;
        if (b < 0 || p < min_priority) return;
    } else if (b < 0) {
        return;
    }
    memb[v] = b;
    atomicAdd(&counts[0], 1);
    if (b >= n) atomicAdd(&counts[1], 1);
}

__global__ void totals_kernel(int64_t n, int L, const int32_t* __restrict__ memb, const int64_t* __restrict__ k,
                              unsigned long long* K, int32_t* size) {
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= n) return;
    const int64_t c = memb[v];
    for (int l = 0; l < L; ++l) atomicAdd(&K[c * L + l], (unsigned long long)k[v * L + l]);
    if (size) atomicAdd(&size[c], 1);
}

__global__ void segment_sum_kernel(int64_t n, const int64_t* __restrict__ seg, const int64_t* __restrict__ w,
                                   unsigned long long* out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) atomicAdd(&out[seg[i]], (unsigned long long)w[i]);
}

__global__ void internal_kernel(int64_t n, const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                                const int64_t* __restrict__ w, const int32_t* __restrict__ memb,
                                unsigned long long* out) {
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= n) return;
    const int32_t c = memb[v];
    long long s = 0;
    for (int64_t e = indptr[v]; e < indptr[v + 1]; ++e)
        if (memb[indices[e]] == c) s += w[e];
    if (s) atomicAdd(out, (unsigned long long)s);
}

static unsigned blocks(int64_t n) { return (unsigned)((n + kThreads - 1) / kThreads); }

}  // namespace leiden
}  // namespace mub

using namespace mub::leiden;

extern "C" {

int mub_leiden_scan(int32_t mode, const int64_t* indptr, const int32_t* indices, const int64_t* w, const int64_t* k,
                    int64_t n, int32_t n_layers, double ce, const double* cl_h, const int32_t* memb,
                    const int32_t* parent, const int64_t* K, const int32_t* size, uint64_t key, int32_t* target,
                    double* gain, int32_t* flags, const int32_t* hubs, int64_t n_hubs, const int64_t* hub_off,
                    const int32_t* hub_slots, int32_t* hub_keys, void* hub_vals, int32_t* hub_lists,
                    int32_t* hub_counts, mub_stream_t stream) {
    MUB_REQUIRE(mode == 0 || mode == 1, "leiden_scan: mode %d", mode);
    MUB_REQUIRE(n_layers >= 1 && n_layers <= MUB_LEIDEN_MAX_LAYERS, "leiden_scan: %d layers", n_layers);
    MUB_REQUIRE(n >= 1 && n < 0x3fffffffLL, "leiden_scan: %lld vertices", (long long)n);
    MUB_REQUIRE(cl_h && memb && K && size && target && gain && flags && (mode == 0 || parent),
                "leiden_scan: null pointer");
    MUB_REQUIRE(n_hubs == 0 || (hubs && hub_off && hub_slots && hub_keys && hub_vals && hub_lists && hub_counts),
                "leiden_scan: hub rows need a workspace");
    Problem P{indptr, indices, w, k, n, n_layers, ce, {0.0, 0.0, 0.0, 0.0}};
    for (int l = 0; l < n_layers; ++l) P.cl[l] = cl_h[l];
    State S{memb, parent, K, size, key, target, gain, flags};
    cudaStream_t st = (cudaStream_t)stream;
    int64_t want = (n + kWarps - 1) / kWarps, cap = (int64_t)mub::sm_count() * 16;
    const unsigned grid = (unsigned)(want < cap ? want : cap);
    if (mode == 0)
        scan_kernel<0><<<grid, kWarps * 32, 0, st>>>(P, S);
    else
        scan_kernel<1><<<grid, kWarps * 32, 0, st>>>(P, S);
    int rc = mub::check_launch("leiden_scan");
    if (rc || n_hubs == 0) return rc;
    const unsigned hgrid = (unsigned)((n_hubs + kWarps - 1) / kWarps);
    auto* vals = (unsigned long long*)hub_vals;
    if (mode == 0)
        scan_hub_kernel<0><<<hgrid, kWarps * 32, 0, st>>>(P, S, hubs, n_hubs, hub_off, hub_slots, hub_keys, vals,
                                                          hub_lists, hub_counts);
    else
        scan_hub_kernel<1><<<hgrid, kWarps * 32, 0, st>>>(P, S, hubs, n_hubs, hub_off, hub_slots, hub_keys, vals,
                                                          hub_lists, hub_counts);
    return mub::check_launch("leiden_scan_hub");
}

int32_t mub_leiden_max_shared_degree(void) { return kMaxDeg; }

int mub_leiden_apply(int32_t mode, int64_t n, int32_t* memb, const int32_t* target, uint64_t key,
                     uint64_t min_priority, void* prio, int32_t* counts, mub_stream_t stream) {
    MUB_REQUIRE(n >= 1 && memb && target && counts && (mode == 1 || prio), "leiden_apply: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    cudaMemsetAsync(counts, 0, 2 * sizeof(int32_t), st);
    apply_kernel<<<blocks(n), kThreads, 0, st>>>(mode, n, memb, target, key, (unsigned long long)min_priority,
                                                 (unsigned long long*)prio, counts);
    return mub::check_launch("leiden_apply");
}

int mub_leiden_totals(int64_t n, int32_t n_layers, const int32_t* memb, const int64_t* k, int64_t n_comm, int64_t* K,
                      int32_t* size, mub_stream_t stream) {
    MUB_REQUIRE(n >= 1 && n_layers >= 1 && n_layers <= MUB_LEIDEN_MAX_LAYERS && memb && k && K,
                "leiden_totals: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    cudaMemsetAsync(K, 0, sizeof(int64_t) * (size_t)n_comm * n_layers, st);
    if (size) cudaMemsetAsync(size, 0, sizeof(int32_t) * (size_t)n_comm, st);
    totals_kernel<<<blocks(n), kThreads, 0, st>>>(n, n_layers, memb, k, (unsigned long long*)K, size);
    return mub::check_launch("leiden_totals");
}

int mub_leiden_segment_sum(int64_t n, const int64_t* seg, const int64_t* w, int64_t n_seg, int64_t* out,
                           mub_stream_t stream) {
    MUB_REQUIRE(n >= 0 && n_seg >= 0 && out, "leiden_segment_sum: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    cudaMemsetAsync(out, 0, sizeof(int64_t) * (size_t)n_seg, st);
    if (n == 0) return mub::check_launch("leiden_segment_sum");
    segment_sum_kernel<<<blocks(n), kThreads, 0, st>>>(n, seg, w, (unsigned long long*)out);
    return mub::check_launch("leiden_segment_sum");
}

int mub_leiden_internal(int64_t n, const int64_t* indptr, const int32_t* indices, const int64_t* w,
                        const int32_t* memb, int64_t* out, mub_stream_t stream) {
    MUB_REQUIRE(n >= 1 && indptr && indices && w && memb && out, "leiden_internal: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    cudaMemsetAsync(out, 0, sizeof(int64_t), st);
    internal_kernel<<<blocks(n), kThreads, 0, st>>>(n, indptr, indices, w, memb, (unsigned long long*)out);
    return mub::check_launch("leiden_internal");
}

}  // extern "C"
