// Differential accessibility: the per-(group, peak) statistics behind scanpy's rank_genes_groups (t-test, Wilcoxon),
// called by muon's rank_peaks_groups (muon/_atac/tools.py:337-373).
//
// stats : one CTA per transposed row (peak).  The row's stored non-zero entries of ranked cells are loaded as
//         (order-preserving value key, 16-bit group code) and sorted by (key, code) with a bitonic network.  One sweep
//         over the sorted entries gives every group its rank sum (or, against a reference group, its Mann-Whitney
//         count against that group) and the tie terms sum(t^3 - t), all in exact integer arithmetic.  The implicit
//         zeros are one tie block whose size per group is n_g - stored_g; it is never materialised, and negative
//         stored values rank below it.  A second sort by (code, key) makes each group's entries one run in ascending
//         value order, and a warp sums each run in a fixed order: the moments do not depend on the order in which the
//         transposition placed the entries, so two calls are bit-identical.
//         Rows that fit in shared memory are sorted there (the host launches one size class at a time).  Longer rows
//         are sorted in a per-CTA slice of a global workspace: every chunk of kChunk entries is sorted in shared
//         memory, the network's strides >= kChunk run in global memory, the rest again chunk by chunk in shared
//         memory.  Both paths run the same network on the same keys, so a row gives the same bits on either.
// score : one thread per (group, peak): Welch's t with p = I_{df/(df+t^2)}(df/2, 1/2), or the Wilcoxon z with
//         p = erfc(|z|/sqrt 2); log fold changes and the fractions of cells with a stored non-zero.
#include <math.h>

#include "common.cuh"

namespace mub {

constexpr int kRankThreads = 512;
constexpr int kRankWarps = kRankThreads / 32;
constexpr uint16_t kNoCode = 0xffffu;          // padding of the sort (sorts after every real code)

template <typename V> struct KeyOf;
template <> struct KeyOf<float> { using T = uint32_t; };
template <> struct KeyOf<double> { using T = unsigned long long; };

// shared-memory entry capacity per value type (the largest short-row class, and the chunk of the long-row sort)
template <typename V> constexpr int kRankCap = sizeof(V) == 4 ? 16384 : 8192;

__device__ __forceinline__ uint32_t order_key(float v) {
    const uint32_t b = __float_as_uint(v);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ unsigned long long order_key(double v) {
    const unsigned long long b = (unsigned long long)__double_as_longlong(v);
    return (b >> 63) ? ~b : (b | (1ull << 63));
}
__device__ __forceinline__ float key_value(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
__device__ __forceinline__ double key_value(unsigned long long k) {
    return __longlong_as_double((long long)((k >> 63) ? (k & ~(1ull << 63)) : ~k));
}
// x^2 rounded in the input's precision, as scanpy squares the stored values before its float64 sum
__device__ __forceinline__ double square_in(float x) { return (double)(x * x); }
__device__ __forceinline__ double square_in(double x) { return x * x; }

__device__ __forceinline__ unsigned long long tie3(unsigned long long t) { return t * t * t - t; }

template <bool BY_CODE, typename K>
__device__ __forceinline__ bool before(K ka, uint16_t ca, K kb, uint16_t cb) {
    if (BY_CODE) return ca < cb || (ca == cb && ka < kb);
    return ka < kb || (ka == kb && ca < cb);
}

// one compare-exchange step (merge size k, stride j) over n entries whose first has network index base
template <bool BY_CODE, typename K>
__device__ void bitonic_step(K* key, uint16_t* code, int n, int64_t base, int64_t k, int j) {
    for (int p = threadIdx.x; p < (n >> 1); p += blockDim.x) {
        const int i = ((p & ~(j - 1)) << 1) | (p & (j - 1));
        const int l = i + j;
        const bool up = ((base + i) & k) == 0;
        const K ki = key[i], kl = key[l];
        const uint16_t ci = code[i], cl = code[l];
        if (up ? before<BY_CODE>(kl, cl, ki, ci) : before<BY_CODE>(ki, ci, kl, cl)) {
            key[i] = kl; key[l] = ki;
            code[i] = cl; code[l] = ci;
        }
    }
}

// sort key/code[0, P) (P a power of two).  In shared memory when P <= chunk (key == skey); otherwise key/code are global
// and skey/scode a shared chunk buffer of `chunk` entries.
template <bool BY_CODE, typename K>
__device__ void bitonic_sort(K* key, uint16_t* code, int64_t P, K* skey, uint16_t* scode, int chunk) {
    if (key == skey) {
        for (int64_t k = 2; k <= P; k <<= 1)
            for (int j = (int)(k >> 1); j > 0; j >>= 1) {
                bitonic_step<BY_CODE>(key, code, (int)P, 0, k, j);
                __syncthreads();
            }
        return;
    }
    auto in_chunks = [&](int64_t k, int j_hi) {          // strides j_hi..1 of merge size k, chunk by chunk
        for (int64_t c = 0; c < P; c += chunk) {
            for (int i = threadIdx.x; i < chunk; i += blockDim.x) {
                skey[i] = key[c + i];
                scode[i] = code[c + i];
            }
            __syncthreads();
            for (int j = j_hi; j > 0; j >>= 1) {
                bitonic_step<BY_CODE>(skey, scode, chunk, c, k, j);
                __syncthreads();
            }
            for (int i = threadIdx.x; i < chunk; i += blockDim.x) {
                key[c + i] = skey[i];
                code[c + i] = scode[i];
            }
            __syncthreads();
        }
    };
    for (int64_t c = 0; c < P; c += chunk) {             // every chunk sorted (merge sizes <= chunk)
        for (int i = threadIdx.x; i < chunk; i += blockDim.x) {
            skey[i] = key[c + i];
            scode[i] = code[c + i];
        }
        __syncthreads();
        for (int64_t k = 2; k <= chunk; k <<= 1)
            for (int j = (int)(k >> 1); j > 0; j >>= 1) {
                bitonic_step<BY_CODE>(skey, scode, chunk, c, k, j);
                __syncthreads();
            }
        for (int i = threadIdx.x; i < chunk; i += blockDim.x) {
            key[c + i] = skey[i];
            code[c + i] = scode[i];
        }
        __syncthreads();
    }
    for (int64_t k = 2 * (int64_t)chunk; k <= P; k <<= 1) {
        for (int64_t j = k >> 1; j >= chunk; j >>= 1) {   // strides that cross chunks: in global memory
            for (int64_t p = threadIdx.x; p < (P >> 1); p += blockDim.x) {
                const int64_t i = ((p & ~(j - 1)) << 1) | (p & (j - 1));
                const int64_t l = i + j;
                const bool up = (i & k) == 0;
                const K ki = key[i], kl = key[l];
                const uint16_t ci = code[i], cl = code[l];
                if (up ? before<BY_CODE>(kl, cl, ki, ci) : before<BY_CODE>(ki, ci, kl, cl)) {
                    key[i] = kl; key[l] = ki;
                    code[i] = cl; code[l] = ci;
                }
            }
            __syncthreads();
        }
        in_chunks(k, chunk >> 1);
    }
}

// first index in [0, m) whose (key, code) is not before (k, c) in (key, code) order
template <typename K>
__device__ __forceinline__ int lower_pair(const K* key, const uint16_t* code, int m, K k, uint16_t c) {
    int lo = 0, hi = m;
    while (lo < hi) {
        const int mid = (int)(((unsigned)lo + (unsigned)hi) >> 1);
        if (before<false>(key[mid], code[mid], k, c)) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}
template <typename K>
__device__ __forceinline__ int upper_key(const K* key, int m, K k) {
    int lo = 0, hi = m;
    while (lo < hi) {
        const int mid = (int)(((unsigned)lo + (unsigned)hi) >> 1);
        if (!(k < key[mid])) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// exclusive prefix count of code == ref over [0, m] into pre[0..m]
__device__ void prefix_ref(const uint16_t* code, int m, uint16_t ref, int32_t* pre, int* warp_tot) {
    const int per = (m + blockDim.x - 1) / blockDim.x;
    const int a = min(m, (int)threadIdx.x * per), b = min(m, a + per);
    int c = 0;
    for (int i = a; i < b; ++i) c += code[i] == ref;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int x = c;
    for (int d = 1; d < 32; d <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= d) x += y;
    }
    if (lane == 31) warp_tot[warp] = x;
    __syncthreads();
    int off = 0;
    for (int w = 0; w < warp; ++w) off += warp_tot[w];
    int run = off + x - c;
    for (int i = a; i < b; ++i) {
        pre[i] = run;
        run += code[i] == ref;
    }
    if (threadIdx.x == blockDim.x - 1) pre[m] = off + x;
    __syncthreads();
}

// The rows of one launch: rows[i] (a row of the transpose) -> output column cols[i].  SHORT: every row holds at most
// `cap` entries (a power of two) and is sorted in shared memory; otherwise the CTA's workspace slice holds `cap`
// entries (the longest row rounded up to a power of two) and shared memory one chunk of kRankCap.
// stats [5][K][n_out]: stored non-zeros, sum, sum of squares, rank sum (codes < K - 1), tie term.
template <typename V, bool SHORT>
__global__ void __launch_bounds__(kRankThreads)
rank_stats_kernel(const int64_t* __restrict__ t_indptr, const int32_t* __restrict__ t_cells, const V* __restrict__ t_vals,
                  const int32_t* __restrict__ cell_code, const int32_t* __restrict__ rows, const int32_t* __restrict__ cols,
                  int32_t n_rows, int32_t n_out, int32_t K, const int64_t* __restrict__ group_n, int64_t n_ranked,
                  uint32_t flags, int cap, unsigned char* __restrict__ ws, int64_t ws_stride, double* __restrict__ stats) {
    using Key = typename KeyOf<V>::T;
    extern __shared__ __align__(16) unsigned char smem[];
    __shared__ int s_m, warp_tot[kRankWarps];
    __shared__ unsigned long long s_tie;
    const bool rank = flags & MUB_RANK_WILCOXON, vs_ref = flags & MUB_RANK_VS_GROUP;
    const int G = K - 1;                               // tested groups; code G = the other ranked cells
    const int chunk = SHORT ? cap : kRankCap<V>;
    unsigned long long* g_r2 = reinterpret_cast<unsigned long long*>(smem);   // [K] twice the rank sum
    unsigned long long* g_corr = g_r2 + K;                                      // [K] per-group tie terms
    Key* skey = reinterpret_cast<Key*>(g_corr + K);                             // [chunk]
    int32_t* g_seg = reinterpret_cast<int32_t*>(skey + chunk);                  // [K + 1] run of each code
    int32_t* spre = g_seg + K + 1;                                              // [cap + 1] (short rows)
    uint16_t* scode = reinterpret_cast<uint16_t*>(spre + (SHORT ? cap + 1 : 0));   // [chunk]
    Key* key = skey;
    uint16_t* code = scode;
    int32_t* pre = spre;
    if (!SHORT) {
        unsigned char* w = ws + (size_t)blockIdx.x * (size_t)ws_stride;
        key = reinterpret_cast<Key*>(w);
        pre = reinterpret_cast<int32_t*>(key + cap);
        code = reinterpret_cast<uint16_t*>(pre + cap + 1);
    }
    const Key kzero = order_key((V)0);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int r = blockIdx.x; r < n_rows; r += gridDim.x) {
        const int64_t e0 = __ldg(t_indptr + rows[r]), e1 = __ldg(t_indptr + rows[r] + 1);
        for (int k = threadIdx.x; k < K; k += blockDim.x) g_r2[k] = g_corr[k] = 0ull;
        if (threadIdx.x == 0) {
            s_m = 0;
            s_tie = 0ull;
        }
        __syncthreads();
        // ranked cells' stored non-zeros (a stored zero is one of the implicit zeros)
        for (int64_t e = e0 + threadIdx.x; e < e1; e += blockDim.x) {
            const V v = t_vals[e];
            const int c = __ldg(cell_code + t_cells[e]);
            if (c >= 0 && v != (V)0) {
                const int slot = atomicAdd(&s_m, 1);
                key[slot] = order_key(v);
                code[slot] = (uint16_t)c;
            }
        }
        __syncthreads();
        const int m = s_m;
        int64_t P = SHORT ? 1 : chunk;                       // the long-row sort works on whole chunks
        while (P < m) P <<= 1;
        for (int64_t i = m + threadIdx.x; i < P; i += blockDim.x) {
            key[i] = ~(Key)0;
            code[i] = kNoCode;
        }
        __syncthreads();
        int neg = 0, zr = 0;
        if (rank) {
            bitonic_sort<false>(key, code, P, skey, scode, chunk);
            neg = lower_pair(key, code, m, kzero, (uint16_t)0);
            if (vs_ref) {
                prefix_ref(code, m, (uint16_t)G, pre, warp_tot);
                zr = (int)(__ldg(group_n + G) - pre[m]);          // the reference group's zeros
            }
            const int nz = (int)(n_ranked - m);                 // every ranked cell's zero (rest)
            for (int i = threadIdx.x; i < m; i += blockDim.x) {
                const Key ki = key[i];
                const uint16_t ci = code[i];
                const bool block_lead = i == 0 || key[i - 1] != ki;
                const bool run_lead = block_lead || code[i - 1] != ci;
                if (!run_lead) continue;
                const int s = block_lead ? i : lower_pair(key, code, m, ki, (uint16_t)0);
                const int e = upper_key(key, m, ki);
                const bool pos = ki > kzero;
                if (!vs_ref) {
                    if (block_lead) atomicAdd(&s_tie, tie3((unsigned long long)(e - s)));
                    if (ci < G) {
                        const int re = lower_pair(key, code, m, ki, (uint16_t)(ci + 1));
                        const unsigned long long t = (unsigned long long)(re - i);
                        atomicAdd(g_r2 + ci, t * (2ull * (unsigned long long)(s + (pos ? nz : 0)) + (unsigned long long)(e - s) + 1ull));
                    }
                } else {
                    const unsigned long long r_in = (unsigned long long)(e - lower_pair(key, code, m, ki, (uint16_t)G));
                    if (block_lead && r_in) atomicAdd(&s_tie, tie3(r_in));
                    if (ci < G) {
                        const int re = lower_pair(key, code, m, ki, (uint16_t)(ci + 1));
                        const unsigned long long t = (unsigned long long)(re - i);
                        const unsigned long long below = (unsigned long long)pre[s] + (pos ? (unsigned long long)zr : 0ull);
                        atomicAdd(g_r2 + ci, t * (2ull * below + r_in));
                        atomicAdd(g_corr + ci, tie3(t + r_in) - tie3(r_in));
                    }
                }
            }
            __syncthreads();
        }
        // (code, key) order: each code's entries are one run, ascending in value
        bitonic_sort<true>(key, code, P, skey, scode, chunk);
        for (int k = threadIdx.x; k <= K; k += blockDim.x) {
            int lo = 0, hi = m;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (code[mid] < k) lo = mid + 1;
                else hi = mid;
            }
            g_seg[k] = lo;
        }
        __syncthreads();
        const int64_t col = cols[r];
        for (int k = warp; k < K; k += kRankWarps) {         // fixed-order moments of each code's run
            const int a = g_seg[k], b = g_seg[k + 1];
            double s1 = 0.0, s2 = 0.0;
            for (int i = a + lane; i < b; i += 32) {
                const V x = (V)key_value(key[i]);
                s1 += (double)x;
                s2 += square_in(x);
            }
            s1 = warp_sum(s1);
            s2 = warp_sum(s2);
            if (lane == 0) {
                stats[((size_t)0 * K + k) * n_out + col] = (double)(b - a);
                stats[((size_t)1 * K + k) * n_out + col] = s1;
                stats[((size_t)2 * K + k) * n_out + col] = s2;
            }
        }
        // the zero block: its tie term, shared by every group (rest: all zeros; against a group: the group's zeros)
        if (rank && threadIdx.x == 0) s_tie += tie3(vs_ref ? (unsigned long long)zr : (unsigned long long)(n_ranked - m));
        __syncthreads();
        for (int k = threadIdx.x; k < K; k += blockDim.x) {
            double rs = 0.0, tie = 0.0;
            if (rank && k < G) {
                const unsigned long long ng = (unsigned long long)__ldg(group_n + k);
                const unsigned long long z = ng - (unsigned long long)(g_seg[k + 1] - g_seg[k]);   // the group's zeros
                unsigned long long r2 = g_r2[k], t3 = s_tie + g_corr[k];
                if (!vs_ref) {
                    r2 += z * (2ull * (unsigned long long)neg + (unsigned long long)(n_ranked - m) + 1ull);
                } else {   // Mann-Whitney count against the reference, + n_g (n_g + 1) / 2 = rank sum within g and r
                    r2 += z * (2ull * (unsigned long long)pre[neg] + (unsigned long long)zr) + ng * (ng + 1ull);
                    t3 += tie3(z + (unsigned long long)zr) - tie3((unsigned long long)zr);
                }
                rs = 0.5 * (double)r2;                       // exact: an integer below 2^53
                tie = (double)t3;
            }
            stats[((size_t)3 * K + k) * n_out + col] = rs;
            stats[((size_t)4 * K + k) * n_out + col] = tie;
        }
        __syncthreads();
    }
}

// ---- regularized incomplete beta for Student's t ------------------------------------------------------------------
// ln B(a, 1/2).  For a >= 20 from Stirling's series, so the difference lgamma(a) - lgamma(a + 1/2) does not lose
// the digits that two large lgamma values share.
__device__ double stirling_rem(double z) {
    const double r = 1.0 / z, r2 = r * r;
    return r * (1.0 / 12 - r2 * (1.0 / 360 - r2 * (1.0 / 1260 - r2 * (1.0 / 1680 - r2 * (1.0 / 1188)))));
}
__device__ double lbeta_half(double a) {
    const double lsqrtpi = 0.57236494292470008707;     // ln Gamma(1/2)
    if (a < 20.0) return lgamma(a) + lsqrtpi - lgamma(a + 0.5);
    return -0.5 * log(a) - a * log1p(0.5 / a) + 0.5 + stirling_rem(a) - stirling_rem(a + 0.5) + lsqrtpi;
}
// continued fraction of I_x(a, b) (modified Lentz)
__device__ double beta_cf(double a, double b, double x) {
    const double tiny = 1e-300;
    const double qab = a + b, qap = a + 1.0, qam = a - 1.0;
    double c = 1.0, d = 1.0 - qab * x / qap;
    if (fabs(d) < tiny) d = tiny;
    d = 1.0 / d;
    double h = d;
    for (int m = 1; m <= 100000; ++m) {
        const int m2 = 2 * m;
        double aa = m * (b - m) * x / ((qam + m2) * (a + m2));
        d = 1.0 + aa * d;
        if (fabs(d) < tiny) d = tiny;
        c = 1.0 + aa / c;
        if (fabs(c) < tiny) c = tiny;
        d = 1.0 / d;
        h *= d * c;
        aa = -(a + m) * (qab + m) * x / ((a + m2) * (qap + m2));
        d = 1.0 + aa * d;
        if (fabs(d) < tiny) d = tiny;
        c = 1.0 + aa / c;
        if (fabs(c) < tiny) c = tiny;
        d = 1.0 / d;
        const double del = d * c;
        h *= del;
        if (fabs(del - 1.0) < 1e-16) break;
    }
    return h;
}
// I_x(a, 1/2) for large a, given ln x: DiDonato & Morris's BGRAT (ACM TOMS 18 (1992) 360, eq. 9), Temme's expansion
// in powers of 1/T with T = a - 1/4 and u = -T ln x:
//   I_x(a, b) = Gamma(a + b) / (Gamma(a) T^b) * sum_n p_n J_n(b, u),   J_0 = Gamma(b, u) / Gamma(b) = erfc(sqrt u),
// J_n by the recursion 9.6 (held here multiplied by u^b e^-u / Gamma(b)), p_n by 9.4.  The continued fraction loses
// about a * eps at large a; this series does not, and needs fewer terms the larger a is.
constexpr double kBgratMinA = 300.0;             // df >= 600: the series takes <= ~20 terms up to p ~ 1e-300
constexpr int kBgratTerms = 30;
__device__ double beta_large_a_half(double a, double lx) {
    const double b = 0.5, T = a - 0.25, u = -T * lx;
    if (!(u < 745.0)) return 0.0;                  // below the smallest subnormal (and ln x = -inf)
    const double su = sqrt(u);
    const double h = exp(-u) * su * 0.56418958354775628695;                      // u^b e^-u / Gamma(b)
    const double pre = exp(0.57236494292470008707 - lbeta_half(a) - 0.5 * log(T));   // Gamma(a+1/2) / (Gamma(a) sqrt T)
    double j = erfc(su), s = j;
    double p[kBgratTerms];
    p[0] = 1.0;
    const double lx2 = 0.25 * lx * lx, t4 = 4.0 * T * T;
    double lxp = 1.0, b2n = b, fact = 1.0;        // (ln x / 2)^(2n - 2), b + 2n - 2, (2n + 1)!
    for (int n = 1; n < kBgratTerms; ++n) {
        fact *= (double)(2 * n) * (double)(2 * n + 1);
        double acc = 0.0, fm = 1.0;                 // fm = (2m + 1)!
        for (int m = 1; m < n; ++m) {
            fm *= (double)(2 * m) * (double)(2 * m + 1);
            acc += ((double)m * b - (double)n) * p[n - m] / fm;
        }
        p[n] = acc / (double)n + (b - 1.0) / fact;
        j = (b2n * (b2n + 1.0) * j + (u + b2n + 1.0) * lxp * h) / t4;
        lxp *= lx2;
        b2n += 2.0;
        const double r = p[n] * j;
        s += r;
        if (fabs(r) <= 1e-17 * fabs(s)) break;
    }
    return fmin(1.0, pre * s);
}
// two-sided p of Student's t with df degrees of freedom: I_{df/(df+t^2)}(df/2, 1/2)
__device__ double student_p(double t, double df) {
    if (isnan(t) || isnan(df)) return nan("");
    const double at = fabs(t);
    if (isinf(at)) return 0.0;
    if (at == 0.0) return 1.0;
    const double t2 = t * t;
    const double a = 0.5 * df, b = 0.5;
    if (a >= kBgratMinA) return beta_large_a_half(a, -log1p(t2 / df));
    if (isinf(t2)) {
        // |t| > 1.3e154: p ~ |t|^-df is still far above the smallest double at small df.  ln x from r = sqrt(df) / |t|.
        const double r = sqrt(df) / at, r2 = r * r;
        const double lx = 2.0 * log(r) - log1p(r2);
        return exp(a * lx - b * log1p(r2) - lbeta_half(a)) * beta_cf(a, b, r2 / (1.0 + r2)) / a;
    }
    const double x = df / (df + t2), y = t2 / (df + t2);
    const double lpre = -a * log1p(t2 / df) + b * log(y) - lbeta_half(a);
    if (x < (a + 1.0) / (a + b + 2.0)) return exp(lpre) * beta_cf(a, b, x) / a;
    return 1.0 - exp(lpre) * beta_cf(b, a, y) / b;
}

__device__ __forceinline__ double expm1_base(double x, double log_base) {
    return log_base > 0.0 ? expm1(x * log_base) : expm1(x);
}

__global__ void __launch_bounds__(256)
rank_score_kernel(const double* __restrict__ stats, int32_t K, int32_t n_out, const int64_t* __restrict__ group_n,
                  int64_t n_total, uint32_t flags, double log_base, double* __restrict__ scores, double* __restrict__ pvals,
                  double* __restrict__ lfc, double* __restrict__ pts, double* __restrict__ pts_rest) {
    const int G = K - 1;
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (int64_t)G * n_out) return;
    const int g = (int)(idx / n_out);
    const int64_t p = idx - (int64_t)g * n_out;
    const bool vs_ref = flags & MUB_RANK_VS_GROUP;
    auto S = [&](int q, int k) { return stats[((size_t)q * K + k) * n_out + p]; };
    const double ng = (double)group_n[g];
    const double cnt_g = S(0, g), sum_g = S(1, g), sq_g = S(2, g);
    double nr, cnt_r, sum_r, sq_r;
    if (vs_ref) {
        nr = (double)group_n[G];
        cnt_r = S(0, G); sum_r = S(1, G); sq_r = S(2, G);
    } else {                                         // rest: every cell outside g; totals in code order
        double c = 0.0, s1 = 0.0, s2 = 0.0;
        for (int k = 0; k < K; ++k) {
            if (k == g) continue;
            c += S(0, k); s1 += S(1, k); s2 += S(2, k);
        }
        nr = (double)(n_total - group_n[g]);
        cnt_r = c; sum_r = s1; sq_r = s2;
    }
    const double mean_g = sum_g / ng, mean_r = sum_r / nr;
    const size_t o = (size_t)g * n_out + p;
    if (flags & MUB_RANK_WILCOXON) {
        const double N = vs_ref ? ng + nr : (double)n_total, mm = N - ng;
        double T = 1.0;
        if (flags & MUB_RANK_TIE_CORRECT) T = 1.0 - S(4, g) / (N * N * N - N);
        const double sd = sqrt(T * ng * mm * (N + 1.0) / 12.0);
        double z = (S(3, g) - ng * ((N + 1.0) / 2.0)) / sd;
        if (isnan(z)) z = 0.0;
        scores[o] = z;
        pvals[o] = erfc(fabs(z) * 0.70710678118654752440);
    } else {
        const double var_g = (sq_g / ng - mean_g * mean_g) * (ng / (ng - 1.0));
        const double var_r = (sq_r / nr - mean_r * mean_r) * (nr / (nr - 1.0));
        const double n2 = (flags & MUB_RANK_OVERESTIM_VAR) ? ng : nr;
        const double vn1 = var_g / ng, vn2 = var_r / n2;
        double df = (vn1 + vn2) * (vn1 + vn2) / (vn1 * vn1 / (ng - 1.0) + vn2 * vn2 / (n2 - 1.0));
        if (isnan(df)) df = 1.0;
        const double t = (mean_g - mean_r) / sqrt(vn1 + vn2);
        const double pv = student_p(t, df);
        scores[o] = isnan(t) ? 0.0 : t;
        pvals[o] = isnan(pv) ? 1.0 : pv;
    }
    lfc[o] = log2((expm1_base(mean_g, log_base) + 1e-9) / (expm1_base(mean_r, log_base) + 1e-9));
    pts[o] = cnt_g / ng;
    if (g == 0 && vs_ref) pts[(size_t)G * n_out + p] = cnt_r / nr;
    if (pts_rest) pts_rest[o] = cnt_r / nr;
}

template <typename V>
static size_t stats_smem(int32_t K, int cap, bool is_short) {
    using Key = typename KeyOf<V>::T;
    const int chunk = is_short ? cap : kRankCap<V>;
    return sizeof(unsigned long long) * 2 * K + sizeof(Key) * chunk + sizeof(int32_t) * (K + 1) +
           (is_short ? sizeof(int32_t) * (cap + 1) : 0) + sizeof(uint16_t) * chunk;
}

template <typename V>
static int launch_stats(const int64_t* t_indptr, const int32_t* t_cells, const V* t_vals, const int32_t* cell_code,
                        const int32_t* rows, const int32_t* cols, int32_t n_rows, int32_t n_out, int32_t K,
                        const int64_t* group_n, int64_t n_ranked, uint32_t flags, int32_t cap, void* ws,
                        int64_t ws_bytes, double* stats, mub_stream_t stream) {
    using Key = typename KeyOf<V>::T;
    MUB_REQUIRE(K >= 2 && K <= MUB_RANK_MAX_GROUPS + 1, "rank_stats: K = %d groups + 1 outside [2, %d]", K,
                MUB_RANK_MAX_GROUPS + 1);
    MUB_REQUIRE(n_rows >= 0 && n_out >= 0 && n_ranked >= 0, "rank_stats: negative size");
    MUB_REQUIRE(n_ranked < 2642245, "rank_stats: %lld ranked cells: the exact tie terms need fewer than 2642245",
                (long long)n_ranked);
    MUB_REQUIRE(cap >= 2 && (cap & (cap - 1)) == 0, "rank_stats: cap %d must be a power of two >= 2", cap);
    if (n_rows == 0) return 0;
    MUB_REQUIRE(t_indptr && t_cells && t_vals && cell_code && rows && cols && group_n && stats, "rank_stats: null pointer");
    const bool is_short = cap <= kRankCap<V>;
    const size_t smem = stats_smem<V>(K, cap, is_short);
    cudaStream_t s = (cudaStream_t)stream;
    int grid = n_rows;
    int64_t stride = 0;
    if (!is_short) {
        stride = (int64_t)((sizeof(Key) + sizeof(int32_t) + sizeof(uint16_t)) * (size_t)cap + 16 + 15) & ~15ll;
        MUB_REQUIRE(ws && ws_bytes >= stride, "rank_stats: workspace of %lld B < one slice of %lld B", (long long)ws_bytes,
                    (long long)stride);
        const int64_t slices = ws_bytes / stride;
        grid = (int)(slices < n_rows ? slices : n_rows);
    }
    cudaError_t e;
    if (is_short) {
        e = cudaFuncSetAttribute(rank_stats_kernel<V, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e == cudaSuccess)
            rank_stats_kernel<V, true><<<grid, kRankThreads, smem, s>>>(t_indptr, t_cells, t_vals, cell_code, rows, cols,
                                                                        n_rows, n_out, K, group_n, n_ranked, flags, cap,
                                                                        nullptr, 0, stats);
    } else {
        e = cudaFuncSetAttribute(rank_stats_kernel<V, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e == cudaSuccess)
            rank_stats_kernel<V, false><<<grid, kRankThreads, smem, s>>>(t_indptr, t_cells, t_vals, cell_code, rows, cols,
                                                                         n_rows, n_out, K, group_n, n_ranked, flags, cap,
                                                                         (unsigned char*)ws, stride, stats);
    }
    if (e != cudaSuccess) {
        set_error("rank_stats: %zu B of shared memory: %s", smem, cudaGetErrorString(e));
        return -2;
    }
    return check_launch("rank_stats");
}

}  // namespace mub

extern "C" {

int32_t mub_rank_shared_capacity(int32_t value_bytes) {
    return value_bytes == 8 ? mub::kRankCap<double> : mub::kRankCap<float>;
}

int64_t mub_rank_workspace_slice_bytes(int32_t value_bytes, int32_t cap) {
    const size_t kb = value_bytes == 8 ? 8 : 4;
    return (int64_t)((kb + sizeof(int32_t) + sizeof(uint16_t)) * (size_t)cap + 16 + 15) & ~15ll;
}

int mub_rank_stats_f32(const int64_t* t_indptr, const int32_t* t_cells, const float* t_vals, const int32_t* cell_code,
                       const int32_t* rows, const int32_t* cols, int32_t n_rows, int32_t n_out, int32_t K,
                       const int64_t* group_n, int64_t n_ranked, uint32_t flags, int32_t cap, void* ws, int64_t ws_bytes,
                       double* stats, mub_stream_t stream) {
    return mub::launch_stats<float>(t_indptr, t_cells, t_vals, cell_code, rows, cols, n_rows, n_out, K, group_n, n_ranked,
                                    flags, cap, ws, ws_bytes, stats, stream);
}

int mub_rank_stats_f64(const int64_t* t_indptr, const int32_t* t_cells, const double* t_vals, const int32_t* cell_code,
                       const int32_t* rows, const int32_t* cols, int32_t n_rows, int32_t n_out, int32_t K,
                       const int64_t* group_n, int64_t n_ranked, uint32_t flags, int32_t cap, void* ws, int64_t ws_bytes,
                       double* stats, mub_stream_t stream) {
    return mub::launch_stats<double>(t_indptr, t_cells, t_vals, cell_code, rows, cols, n_rows, n_out, K, group_n, n_ranked,
                                     flags, cap, ws, ws_bytes, stats, stream);
}

int mub_rank_score(const double* stats, int32_t K, int32_t n_out, const int64_t* group_n, int64_t n_total, uint32_t flags,
                   double log_base, double* scores, double* pvals, double* lfc, double* pts, double* pts_rest,
                   mub_stream_t stream) {
    MUB_REQUIRE(K >= 2 && n_out >= 0, "rank_score: bad shape");
    if (n_out == 0) return 0;
    MUB_REQUIRE(stats && group_n && scores && pvals && lfc && pts, "rank_score: null pointer");
    const int64_t n = (int64_t)(K - 1) * n_out;
    mub::rank_score_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        stats, K, n_out, group_n, n_total, flags, log_base, scores, pvals, lfc, pts, pts_rest);
    return mub::check_launch("rank_score");
}

}  // extern "C"
