// Host <-> device staging engine for the ingest side of the hot path (SURVEY section 8 row f2).
//
// The reference keeps AnnData.X as a pageable scipy CSR in host memory (muon/_atac/preproc.py:86-129
// reads adata.X / adata.layers[...] and rebinds a freshly allocated matrix).  A drop-in GPU path
// therefore starts and ends in pageable memory: 72 GB in / 24 GB out at BASELINE configs[1].
// cudaMemcpy from pageable memory runs at a few GB/s, so transfers are staged through a small ring
// of pinned buffers that a pool of host threads fills (H2D) or drains (D2H) while the DMA engine
// works on the previous chunk.  Two things are fused into that copy so that no byte of host memory
// is touched twice:
//   * narrowing of scipy's int64 index arrays (nnz >= 2^31) to the int32 the kernels use,
//   * a position-dependent 64-bit fingerprint of the element stream, which lets a later call
//     prove that a host array still equals its device twin without a device pass.
//
// Pure host code (std::thread + cudaMemcpyAsync); compiled by nvcc with the rest of the library.
#include <atomic>
#include <condition_variable>
#include <cstring>
#include <functional>
#include <mutex>
#include <thread>
#include <vector>

#include "common.cuh"

namespace mub {

// ---- fingerprint of a stream of 32-bit elements e_i, i = 0..n-1:
//        H = sum_i  u64(e_i ^ a_i) * u64(b_i)   mod 2^64,     a_i = u32(i*K1 + hi(i)*K3 + C1),  b_i = u32(i*K2 + hi(i)*K4 + C2) | 1
// Every term carries its position, so partial sums over disjoint ranges just add up (thread- and chunk-order
// independent), while any single-element edit (b_i is odd: x -> x*b_i is injective on 32-bit x) or permutation
// changes the value.  32 x 32 -> 64-bit products only: the host loop vectorises (vpmuludq), the device kernel is
// trivially HBM-bound.  hi(i) = i >> 32 keeps positions beyond 2^32 distinct.
constexpr uint32_t kK1 = 0x9E3779B1u, kK2 = 0x85EBCA6Bu, kK3 = 0xC2B2AE35u, kK4 = 0x27D4EB2Fu, kC1 = 0x7F4A7C15u,
                   kC2 = 0x165667B1u;

__host__ __device__ inline uint64_t hash_term(uint32_t e, uint64_t i) {
    const uint32_t lo = (uint32_t)i, hi = (uint32_t)(i >> 32);
    const uint32_t a = lo * kK1 + hi * kK3 + kC1;
    const uint32_t b = (lo * kK2 + hi * kK4 + kC2) | 1u;
    return (uint64_t)(e ^ a) * (uint64_t)b;
}

// [pos0, pos0 + n) must not cross a multiple of 2^32 (callers split there), so hi(i) is a loop constant
#if defined(__GNUC__) && !defined(__CUDA_ARCH__)
#define MUB_SIMD_CLONES __attribute__((target_clones("avx512f", "avx2", "default")))
#else
#define MUB_SIMD_CLONES
#endif

MUB_SIMD_CLONES static uint64_t hash_run_u32(const uint32_t* src, size_t n, uint64_t pos0) {
    const uint32_t hi = (uint32_t)(pos0 >> 32), lo0 = (uint32_t)pos0;
    const uint32_t abase = hi * kK3 + kC1, bbase = hi * kK4 + kC2;
    uint64_t h = 0;
    for (size_t j = 0; j < n; ++j) {
        const uint32_t lo = lo0 + (uint32_t)j;
        const uint32_t a = lo * kK1 + abase, b = (lo * kK2 + bbase) | 1u;
        h += (uint64_t)(src[j] ^ a) * (uint64_t)b;
    }
    return h;
}

MUB_SIMD_CLONES static uint64_t hash_run_i64(const int64_t* src, size_t n, uint64_t pos0) {
    const uint32_t hi = (uint32_t)(pos0 >> 32), lo0 = (uint32_t)pos0;
    const uint32_t abase = hi * kK3 + kC1, bbase = hi * kK4 + kC2;
    uint64_t h = 0;
    for (size_t j = 0; j < n; ++j) {
        const uint32_t lo = lo0 + (uint32_t)j;
        const uint32_t a = lo * kK1 + abase, b = (lo * kK2 + bbase) | 1u;
        h += (uint64_t)((uint32_t)src[j] ^ a) * (uint64_t)b;
    }
    return h;
}

// float32 -> uint8 for count data (peak counts are "mostly 1 and 2"): a quarter of the bytes on the bus.  Returns
// non-zero if some value is not an integer in [0, 255] (the caller then sends the block as it is).
MUB_SIMD_CLONES static int narrow_f32_u8(uint8_t* dst, const float* src, size_t n) {
    // branch-free so that it vectorises (cvttps2dq / cvtdq2ps / compare / pack): a float that is not an integer in
    // [0, 255] either fails the round trip or leaves bits above the low byte (NaN and out-of-range values convert to
    // INT_MIN on x86)
    int bad = 0;
    for (size_t i = 0; i < n; ++i) {
        const float v = src[i];
        const int iv = (int)v;
        bad |= ((float)iv != v) | (iv & ~255);
        dst[i] = (uint8_t)iv;
    }
    return bad != 0;
}

static uint64_t hash_only(const void* src, size_t n, int elem_bytes, uint64_t pos0) {
    uint64_t h = 0;
    size_t done = 0;
    while (done < n) {                                    // split at multiples of 2^32
        const uint64_t p = pos0 + done;
        const uint64_t room = ((p >> 32) + 1) * (1ull << 32) - p;
        const size_t m = (n - done) < room ? (n - done) : (size_t)room;
        h += elem_bytes == 8 ? hash_run_i64((const int64_t*)src + done, m, p) : hash_run_u32((const uint32_t*)src + done, m, p);
        done += m;
    }
    return h;
}

// int64 -> int32 narrowing of one run (vectorises); returns non-zero if a value does not fit
MUB_SIMD_CLONES static int narrow_i64(int32_t* dst, const int64_t* src, size_t n) {
    int64_t bad = 0;
    for (size_t i = 0; i < n; ++i) {
        const int64_t v = src[i];
        dst[i] = (int32_t)v;
        bad |= (v ^ (int64_t)(int32_t)v);
    }
    return bad != 0;
}

// ---- a small persistent worker pool: run(fn, parts) executes fn(part) for part in [0, parts) ------
class Pool {
  public:
    explicit Pool(int n) : n_(n < 1 ? 1 : n) {
        for (int t = 0; t < n_ - 1; ++t) threads_.emplace_back([this] { loop(); });
    }
    ~Pool() {
        {
            std::lock_guard<std::mutex> g(m_);
            stop_ = true;
            ++gen_;
        }
        cv_.notify_all();
        for (auto& t : threads_) t.join();
    }
    int size() const { return n_; }
    void run(const std::function<void(int)>& fn, int parts) {
        {
            std::lock_guard<std::mutex> g(m_);
            fn_ = &fn;
            parts_ = parts;
            next_ = 0;
            pending_ = parts;
            ++gen_;
        }
        cv_.notify_all();
        work();  // the calling thread takes parts too
        std::unique_lock<std::mutex> lk(m_);
        done_.wait(lk, [this] { return pending_ == 0; });
        fn_ = nullptr;
        parts_ = next_ = 0;
    }

  private:
    // every piece of shared state is read and written under m_ (a run hands out at most a few dozen parts,
    // each worth >= 100 us of copying, so the lock is never contended for long)
    void work() {
        for (;;) {
            const std::function<void(int)>* fn;
            int p;
            {
                std::lock_guard<std::mutex> g(m_);
                if (fn_ == nullptr || next_ >= parts_) return;
                p = next_++;
                fn = fn_;
            }
            (*fn)(p);
            std::lock_guard<std::mutex> g(m_);
            if (--pending_ == 0) done_.notify_all();
        }
    }
    void loop() {
        uint64_t seen = 0;
        for (;;) {
            {
                std::unique_lock<std::mutex> lk(m_);
                cv_.wait(lk, [&] { return gen_ != seen; });
                seen = gen_;
                if (stop_) return;
            }
            work();
        }
    }
    int n_;
    std::vector<std::thread> threads_;
    std::mutex m_;
    std::condition_variable cv_, done_;
    const std::function<void(int)>* fn_ = nullptr;
    int parts_ = 0, pending_ = 0;
    int next_ = 0;
    uint64_t gen_ = 0;
    bool stop_ = false;
};

struct Stager {
    size_t buf_bytes = 0;       // bytes per ring buffer
    int n_bufs = 0;
    int device = 0;             // CUDA device the ring and the events belong to
    std::vector<void*> bufs;    // the ring is used as n_threads x 2 private sub-buffers (see stage_of)
    std::vector<cudaEvent_t> events;   // one per (thread, sub-buffer)
    Pool* pool = nullptr;
    size_t sub_bytes = 0;

    // sub-buffer j (0/1) of worker t: the ring is one logical array of n_bufs * buf_bytes bytes cut into 2T pieces
    char* stage_of(int t, int j) const {
        const size_t idx = (size_t)(2 * t + j) * sub_bytes;
        return (char*)bufs[idx / buf_bytes] + idx % buf_bytes;
    }
};

#define MUB_CUDA(call, what)                                          \
    do {                                                              \
        cudaError_t e_ = (call);                                      \
        if (e_ != cudaSuccess) {                                      \
            mub::set_error("%s: %s", what, cudaGetErrorString(e_));   \
            return -2;                                                \
        }                                                             \
    } while (0)

}  // namespace mub

extern "C" {

int mub_stager_create(size_t buf_bytes, int32_t n_bufs, int32_t n_threads, void** out) {
    MUB_REQUIRE(out != nullptr, "stager_create: null out");
    // n_bufs == 0: thread pool only (host fingerprints; needs no CUDA context)
    MUB_REQUIRE(buf_bytes >= 4096 && (buf_bytes % 4096) == 0 && (n_bufs == 0 || (n_bufs >= 2 && n_bufs <= 64)) && n_threads >= 1,
                "stager_create: need buf_bytes >= 4096 (multiple of 4096), 0 or 2..64 buffers, >=1 thread");
    auto* s = new mub::Stager();
    s->buf_bytes = buf_bytes;
    s->n_bufs = n_bufs;
    if (n_bufs > 0) {
        cudaGetDevice(&s->device);
        // every worker owns two sub-buffers; a sub-buffer must not straddle two ring buffers
        size_t sub = (buf_bytes * (size_t)n_bufs) / (2 * (size_t)n_threads);
        sub &= ~(size_t)4095;
        while (sub >= 4096 && (buf_bytes % sub) != 0) sub -= 4096;
        if (sub < 4096) {
            mub::set_error("stager_create: %d threads need a larger staging ring than %zu bytes", n_threads, buf_bytes * n_bufs);
            delete s;
            return -1;
        }
        s->sub_bytes = sub;
    }
    for (int i = 0; i < n_bufs; ++i) {
        void* p = nullptr;
        cudaError_t e = cudaHostAlloc(&p, buf_bytes, cudaHostAllocDefault);
        if (e != cudaSuccess) {
            mub::set_error("stager_create: cudaHostAlloc(%zu): %s", buf_bytes, cudaGetErrorString(e));
            for (void* q : s->bufs) cudaFreeHost(q);
            delete s;
            return -2;
        }
        s->bufs.push_back(p);
    }
    if (n_bufs > 0)
        for (int i = 0; i < 2 * n_threads; ++i) {
            cudaEvent_t ev;
            cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
            s->events.push_back(ev);
        }
    s->pool = new mub::Pool(n_threads);
    *out = s;
    return 0;
}

int mub_stager_destroy(void* handle) {
    if (!handle) return 0;
    auto* s = (mub::Stager*)handle;
    delete s->pool;
    for (void* p : s->bufs) cudaFreeHost(p);
    for (auto ev : s->events) cudaEventDestroy(ev);
    delete s;
    return 0;
}

// Pageable host -> device.  src_elem_bytes: 1, 4 or 8 (bytes of one source element);  narrow = 1 (8-byte sources):
// int64 -> int32; narrow = 2 (4-byte sources): float32 -> uint8; a value that does not survive sets *overflow_h.
// hash_h (optional): fingerprint of the uploaded stream as 32-bit elements (4-byte sources, or narrow = 1).
// The array is cut into one contiguous slab per worker thread; every worker converts its slab piece by piece into
// its two private pinned sub-buffers and enqueues the DMA of each piece on `stream` itself (the runtime API is
// thread-safe; copies of different workers interleave on the stream).  One wake-up of the pool per CALL -- an
// earlier version synchronised the pool once per 64 MB chunk.  Returns when the last piece is enqueued.
int mub_stager_h2d(void* handle, const void* src_h, void* dst, size_t n_elems, int32_t src_elem_bytes, int32_t narrow,
                   uint64_t* hash_h, int32_t* overflow_h, mub_stream_t stream) {
    using namespace mub;
    MUB_REQUIRE(handle != nullptr && ((mub::Stager*)handle)->n_bufs >= 2, "stager_h2d: stager has no staging buffers");
    MUB_REQUIRE(src_elem_bytes == 4 || src_elem_bytes == 8 || src_elem_bytes == 1, "stager_h2d: element size must be 1, 4 or 8");
    MUB_REQUIRE(narrow == 0 || (narrow == 1 && src_elem_bytes == 8) || (narrow == 2 && src_elem_bytes == 4),
                "stager_h2d: narrow = 1 (int64 -> int32) needs 8-byte, narrow = 2 (float32 -> uint8) 4-byte source elements");
    MUB_REQUIRE(!hash_h || (src_elem_bytes == 4 && narrow == 0) || narrow == 1, "stager_h2d: fingerprint needs 32-bit elements");
    if (hash_h) *hash_h = 0;
    if (n_elems == 0) return 0;
    MUB_REQUIRE(src_h && dst, "stager_h2d: null pointer");
    auto* s = (Stager*)handle;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t dst_elem = narrow == 1 ? 4 : (narrow == 2 ? 1 : (size_t)src_elem_bytes);
    const int T = s->pool->size();
    // slabs of whole 64-element groups; small arrays use fewer workers
    size_t groups = (n_elems + 63) / 64;
    int workers = (int)(groups < (size_t)T * 1024 ? (groups + 1023) / 1024 : T);
    if (workers < 1) workers = 1;
    const size_t slab = ((groups + workers - 1) / workers) * 64;
    const size_t per_piece = s->sub_bytes / dst_elem;   // elements per sub-buffer (the staged, converted form)
    std::vector<uint64_t> partial(workers, 0);
    std::atomic<int> overflow{0}, failed{0};
    std::function<void(int)> fn = [&](int t) {
        cudaSetDevice(s->device);
        const size_t lo = (size_t)t * slab, hi = lo + slab < n_elems ? lo + slab : n_elems;
        uint64_t h = 0;
        int j = 0;
        for (size_t off = lo; off < hi; off += per_piece, j ^= 1) {
            const size_t cnt = hi - off < per_piece ? hi - off : per_piece;
            char* stage = s->stage_of(t, j);
            if (cudaEventSynchronize(s->events[2 * t + j]) != cudaSuccess) { failed = 1; return; }
            const char* src = (const char*)src_h + off * (size_t)src_elem_bytes;
            if (narrow == 1) {
                if (narrow_i64((int32_t*)stage, (const int64_t*)src, cnt)) overflow = 1;
            } else if (narrow == 2) {
                if (narrow_f32_u8((uint8_t*)stage, (const float*)src, cnt)) overflow = 1;
            } else {
                memcpy(stage, src, cnt * (size_t)src_elem_bytes);
            }
            if (hash_h) h += hash_only(stage, cnt, 4, off);
            if (cudaMemcpyAsync((char*)dst + off * dst_elem, stage, cnt * dst_elem, cudaMemcpyHostToDevice, st) != cudaSuccess ||
                cudaEventRecord(s->events[2 * t + j], st) != cudaSuccess) { failed = 1; return; }
        }
        partial[t] = h;
    };
    s->pool->run(fn, workers);
    if (failed.load()) {
        cudaError_t e = cudaGetLastError();
        set_error("stager_h2d: %s", cudaGetErrorString(e));
        return -2;
    }
    if (hash_h) {
        uint64_t h = 0;
        for (int t = 0; t < workers; ++t) h += partial[t];
        *hash_h = h;
    }
    if (overflow_h && overflow.load()) *overflow_h = 1;
    return 0;
}

// Device -> pageable host, n_bytes (multiple of 4 when a fingerprint is requested).  Synchronous with respect to
// the host: returns when dst_h is complete.  Same slab-per-worker scheme as mub_stager_h2d, each worker
// double-buffered: the DMA of its next piece runs while it copies the previous one out of pinned memory.
int mub_stager_d2h(void* handle, const void* src, void* dst_h, size_t n_bytes, uint64_t* hash_h, mub_stream_t stream) {
    using namespace mub;
    MUB_REQUIRE(handle != nullptr && ((mub::Stager*)handle)->n_bufs >= 2, "stager_d2h: stager has no staging buffers");
    MUB_REQUIRE(!hash_h || (n_bytes % 4) == 0, "stager_d2h: fingerprint needs a multiple of 4 bytes");
    if (hash_h) *hash_h = 0;
    if (n_bytes == 0) return 0;
    MUB_REQUIRE(src && dst_h, "stager_d2h: null pointer");
    auto* s = (Stager*)handle;
    cudaStream_t st = (cudaStream_t)stream;
    const int T = s->pool->size();
    size_t groups = (n_bytes + 4095) / 4096;
    int workers = (int)(groups < (size_t)T * 64 ? (groups + 63) / 64 : T);
    if (workers < 1) workers = 1;
    const size_t slab = ((groups + workers - 1) / workers) * 4096;
    const size_t per_piece = s->sub_bytes;
    std::vector<uint64_t> partial(workers, 0);
    std::atomic<int> failed{0};
    std::function<void(int)> fn = [&](int t) {
        cudaSetDevice(s->device);
        const size_t lo = (size_t)t * slab, hi = lo + slab < n_bytes ? lo + slab : n_bytes;
        if (lo >= hi) return;
        auto issue = [&](size_t off, int j) -> bool {
            const size_t cnt = hi - off < per_piece ? hi - off : per_piece;
            // an earlier transfer (possibly on another stream) may still read this sub-buffer
            return cudaEventSynchronize(s->events[2 * t + j]) == cudaSuccess &&
                   cudaMemcpyAsync(s->stage_of(t, j), (const char*)src + off, cnt, cudaMemcpyDeviceToHost, st) == cudaSuccess &&
                   cudaEventRecord(s->events[2 * t + j], st) == cudaSuccess;
        };
        uint64_t h = 0;
        int j = 0;
        if (!issue(lo, 0)) { failed = 1; return; }
        for (size_t off = lo; off < hi; off += per_piece, j ^= 1) {
            const size_t cnt = hi - off < per_piece ? hi - off : per_piece;
            if (off + per_piece < hi && !issue(off + per_piece, j ^ 1)) { failed = 1; return; }
            if (cudaEventSynchronize(s->events[2 * t + j]) != cudaSuccess) { failed = 1; return; }
            memcpy((char*)dst_h + off, s->stage_of(t, j), cnt);
            if (hash_h) h += hash_only(s->stage_of(t, j), cnt / 4, 4, off / 4);
        }
        partial[t] = h;
    };
    s->pool->run(fn, workers);
    if (failed.load()) {
        cudaError_t e = cudaGetLastError();
        set_error("stager_d2h: %s", cudaGetErrorString(e));
        return -2;
    }
    if (hash_h) {
        uint64_t h = 0;
        for (int t = 0; t < workers; ++t) h += partial[t];
        *hash_h = h;
    }
    return 0;
}

// Fingerprint of a host array without copying it: n_elems elements of 4 bytes, or of 8 bytes read as int64 and
// narrowed to int32 (so that a host int64 index array and its int32 device twin have the same fingerprint).
int mub_host_fingerprint(void* handle, const void* src_h, size_t n_elems, int32_t elem_bytes, uint64_t* hash_h) {
    using namespace mub;
    MUB_REQUIRE(handle && hash_h, "host_fingerprint: null pointer");
    MUB_REQUIRE(elem_bytes == 4 || elem_bytes == 8, "host_fingerprint: element size must be 4 or 8");
    *hash_h = 0;
    if (n_elems == 0) return 0;
    MUB_REQUIRE(src_h, "host_fingerprint: null source");
    auto* s = (Stager*)handle;
    const int T = s->pool->size();
    const size_t block = (size_t)1 << 20;                      // elements per work item
    const size_t n_blocks = (n_elems + block - 1) / block;
    std::vector<uint64_t> partial(T, 0);
    std::atomic<size_t> next{0};
    std::function<void(int)> fn = [&](int p) {
        uint64_t h = 0;
        for (;;) {
            const size_t bi = next.fetch_add(1);
            if (bi >= n_blocks) break;
            const size_t i0 = bi * block;
            const size_t m = n_elems - i0 < block ? n_elems - i0 : block;
            h += hash_only((const char*)src_h + i0 * (size_t)elem_bytes, m, elem_bytes, i0);
        }
        partial[p] = h;
    };
    s->pool->run(fn, T);
    uint64_t h = 0;
    for (int p = 0; p < T; ++p) h += partial[p];
    *hash_h = h;
    return 0;
}

}  // extern "C"

namespace mub {
__global__ void __launch_bounds__(256)
fingerprint_kernel(const uint32_t* __restrict__ src, int64_t n, unsigned long long* out) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    uint64_t h = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        h += hash_term((uint32_t)ld_stream((const int*)src + i), (uint64_t)i);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) h += __shfl_xor_sync(0xffffffffu, h, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(out, (unsigned long long)h);
}
}  // namespace mub

namespace mub {
__global__ void __launch_bounds__(256)
u8_to_f32_kernel(const uchar4* __restrict__ src, int64_t n4, float4* __restrict__ dst) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        const uchar4 v = src[i];
        dst[i] = make_float4((float)v.x, (float)v.y, (float)v.z, (float)v.w);
    }
}
__global__ void u8_to_f32_tail_kernel(const uint8_t* __restrict__ src, int64_t n, float* __restrict__ dst) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = (float)src[i];
}
}  // namespace mub

// dst[i] = (float)src[i]: widens count data that crossed the bus as uint8 (mub_stager_h2d narrow = 2)
extern "C" int mub_u8_to_f32(const void* src, int64_t n, float* dst, mub_stream_t stream) {
    MUB_REQUIRE(n >= 0, "u8_to_f32: negative size");
    if (n == 0) return 0;
    MUB_REQUIRE(src && dst, "u8_to_f32: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    const bool vec = (((uintptr_t)src & 3) == 0) && (((uintptr_t)dst & 15) == 0);
    const int64_t n4 = vec ? n / 4 : 0;
    if (n4 > 0) {
        int64_t want = (n4 + 255) / 256, cap = (int64_t)mub::sm_count() * 8;
        mub::u8_to_f32_kernel<<<(int)(want < cap ? want : cap), 256, 0, s>>>((const uchar4*)src, n4, (float4*)dst);
    }
    const int64_t rest = n - 4 * n4;
    if (rest > 0)
        mub::u8_to_f32_tail_kernel<<<(int)((rest + 255) / 256), 256, 0, s>>>((const uint8_t*)src + 4 * n4, rest, dst + 4 * n4);
    return mub::check_launch("u8_to_f32");
}

// Same fingerprint of a device array of n 32-bit elements, ACCUMULATED into *out (device uint64, zero it first).
extern "C" int mub_device_fingerprint(const void* src, int64_t n, uint64_t* out, mub_stream_t stream) {
    MUB_REQUIRE(n >= 0 && out, "device_fingerprint: bad argument");
    if (n == 0) return 0;
    MUB_REQUIRE(src, "device_fingerprint: null source");
    int64_t want = (n + 255) / 256, cap = (int64_t)mub::sm_count() * 8;
    int grid = (int)(want < cap ? want : cap);
    mub::fingerprint_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const uint32_t*)src, n, (unsigned long long*)out);
    return mub::check_launch("device_fingerprint");
}
