// K2 v2 -- CSR x dense SpMM with the dense operand staged through shared memory by TMA.
//
// The v1 row-warp kernel (spmm.cu) gathers 4P bytes of B per non-zero straight from L2, with almost
// no L1 reuse.  Here a persistent CTA owns a block
// of R = 32*warps rows and sweeps the COLUMN axis in panels: panel p of B (panel_cols x P floats,
// contiguous in row-major B) is copied into shared memory by one cp.async.bulk (TMA) per panel,
// double-buffered behind mbarriers, and every row of the block consumes its non-zeros whose
// column falls inside the panel from shared memory.  Accumulators for all 32 rows of a warp live
// in registers for the whole sweep (lane l holds columns [l*P/32, (l+1)*P/32) of each row), so B
// traffic from L2 drops by ~R*density*... = (non-zeros per row-block and panel) / panel_cols.
//
// Requires column indices sorted within each row (canonical CSR): a row's entries inside a panel
// are then a contiguous run found by a per-row cursor (lane r of each warp keeps row r's cursor).
// Summation order per row = column order, sequential: deterministic, same as scipy's csr_matvec.
#include "common.cuh"

namespace mub {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes));
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t done = 0;
    while (!done) {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n"
            : "=r"(done)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    }
}
// TMA 1-D bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void tma_bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

template <int P>
struct PanelCfg {
    static constexpr int VEC = P / 32;                          // floats per lane per row
    static constexpr int THREADS = (P == 128) ? 256 : 512;      // accumulators: 32*VEC regs per lane
    static constexpr int WARPS = THREADS / 32;
    static constexpr int ROWS = WARPS * 32;                     // rows per CTA block
};

// explicit shared-space loads (32-bit addresses): keeps the inner loop on LDS instead of generic LD
__device__ __forceinline__ int4 lds_v4(uint32_t addr) {
    int4 r;
    asm volatile("ld.shared.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(addr));
    return r;
}
template <int VEC>
__device__ __forceinline__ void fma_lds(float (&acc)[VEC], float v, uint32_t addr) {
    if constexpr (VEC == 1) {
        float b;
        asm volatile("ld.shared.f32 %0, [%1];" : "=f"(b) : "r"(addr));
        acc[0] = fmaf(v, b, acc[0]);
    } else if constexpr (VEC == 2) {
        float b0, b1;
        asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(b0), "=f"(b1) : "r"(addr));
        acc[0] = fmaf(v, b0, acc[0]);
        acc[1] = fmaf(v, b1, acc[1]);
    } else {
        float b0, b1, b2, b3;
        asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(b0), "=f"(b1), "=f"(b2), "=f"(b3) : "r"(addr));
        acc[0] = fmaf(v, b0, acc[0]);
        acc[1] = fmaf(v, b1, acc[1]);
        acc[2] = fmaf(v, b2, acc[2]);
        acc[3] = fmaf(v, b3, acc[3]);
    }
}

template <int P>
__global__ void __launch_bounds__(PanelCfg<P>::THREADS, 1)
spmm_csr_panel_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                      const float* __restrict__ data, int64_t n_rows, int32_t n_cols,
                      const float* __restrict__ B, float* __restrict__ C, int accumulate, int panel_cols) {
    using Cfg = PanelCfg<P>;
    constexpr int VEC = Cfg::VEC;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float* buf[2];
    buf[0] = reinterpret_cast<float*>(smem_raw);
    buf[1] = buf[0] + (size_t)panel_cols * P;
    uint64_t* full = reinterpret_cast<uint64_t*>(buf[1] + (size_t)panel_cols * P);
    // per-warp staging of one row segment: 2 x 32 entries of {byte offset of the B row in the panel, value}
    int2* stage_all = reinterpret_cast<int2*>(full + 2);
    const uint32_t buf_u32[2] = {smem_u32(buf[0]), smem_u32(buf[1])};

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n_panels = (n_cols + panel_cols - 1) / panel_cols;
    const int64_t n_blocks = (n_rows + Cfg::ROWS - 1) / Cfg::ROWS;

    if (tid == 0) {
        mbar_init(&full[0], 1);
        mbar_init(&full[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    uint32_t issued = 0;     // panels issued so far by this CTA (thread 0 only uses it)
    uint32_t consumed = 0;   // panels consumed so far (all threads; gives buffer + parity)

    auto issue = [&](int p) {  // thread 0: TMA panel p into buffer (issued & 1)
        const int j0 = p * panel_cols;
        const int cols = (n_cols - j0 < panel_cols) ? (n_cols - j0) : panel_cols;
        const uint32_t bytes = (uint32_t)cols * P * sizeof(float);
        uint64_t* bar = &full[issued & 1];
        mbar_expect_tx(bar, bytes);
        tma_bulk_g2s(buf[issued & 1], B + (size_t)j0 * P, bytes, bar);
        ++issued;
    };

    for (int64_t blk = blockIdx.x; blk < n_blocks; blk += gridDim.x) {
        const int64_t row0 = blk * Cfg::ROWS + (int64_t)warp * 32;
        // lane r keeps the cursor / end of row (row0 + r), relative to the block's first non-zero
        const int64_t blk_first = __ldg(indptr + blk * Cfg::ROWS);
        const int64_t my_row = row0 + lane;
        int cur = 0, end = 0;
        if (my_row < n_rows) {
            cur = (int)(__ldg(indptr + my_row) - blk_first);
            end = (int)(__ldg(indptr + my_row + 1) - blk_first);
        }
        const int32_t* idx = indices + blk_first;
        const float* val = data + blk_first;

        int2* my_stage = stage_all + warp * 64;
        float acc[32][VEC];
#pragma unroll
        for (int r = 0; r < 32; ++r)
#pragma unroll
            for (int e = 0; e < VEC; ++e) acc[r][e] = 0.f;

        if (tid == 0) {  // prologue: two panels in flight
            issue(0);
            if (n_panels > 1) issue(1);
        }
        for (int p = 0; p < n_panels; ++p) {
            const int j0 = p * panel_cols;
            const int j1 = (j0 + panel_cols < n_cols) ? j0 + panel_cols : n_cols;
            const uint32_t panel = buf_u32[consumed & 1] + lane * VEC * 4;
            mbar_wait(&full[consumed & 1], (consumed >> 1) & 1);

            // software pipeline over groups of G rows: the first 32 candidates (index, value) of the
            // next G rows are in flight while the current G rows are consumed from registers
            constexpr int G = 8;
            int nc[G];
            float nv[G];
#pragma unroll
            for (int i = 0; i < G; ++i) {
                const int b0 = __shfl_sync(0xffffffffu, cur, i), e0 = __shfl_sync(0xffffffffu, end, i);
                const int k0 = b0 + lane;
                nc[i] = (k0 < e0) ? ld_stream(idx + k0) : 0x7fffffff;
                nv[i] = (k0 < e0) ? ld_stream(val + k0) : 0.f;
            }
#pragma unroll
            for (int g = 0; g < 32 / G; ++g) {
                int cc[G];
                float cv[G];
#pragma unroll
                for (int i = 0; i < G; ++i) { cc[i] = nc[i]; cv[i] = nv[i]; }
                if (g + 1 < 32 / G) {
#pragma unroll
                    for (int i = 0; i < G; ++i) {
                        const int rn = (g + 1) * G + i;
                        const int b0 = __shfl_sync(0xffffffffu, cur, rn), e0 = __shfl_sync(0xffffffffu, end, rn);
                        const int k0 = b0 + lane;
                        nc[i] = (k0 < e0) ? ld_stream(idx + k0) : 0x7fffffff;
                        nv[i] = (k0 < e0) ? ld_stream(val + k0) : 0.f;
                    }
                }
#pragma unroll
                for (int i = 0; i < G; ++i) {
                    const int r = g * G + i;
                    int base = __shfl_sync(0xffffffffu, cur, r);
                    const int rend = __shfl_sync(0xffffffffu, end, r);
                    int c = cc[i];
                    float v = cv[i];
                    for (;;) {
                        const bool inp = c < j1;
                        const unsigned m = __ballot_sync(0xffffffffu, inp);
                        const int cnt = __popc(m);  // sorted row: in-panel entries are a prefix
                        // stage the segment in this warp's shared scratch (zero weight beyond cnt) and read
                        // it back by broadcast: no shuffles, hence no per-shuffle convergence barriers
                        int2* st = my_stage + ((r & 1) << 5);
                        st[lane] = make_int2(inp ? (c - j0) * (P * 4) : 0, inp ? __float_as_int(v) : 0);
                        __syncwarp();
                        const uint32_t st_u32 = smem_u32(st);
                        for (int t = 0; t < cnt; t += 4) {
                            const int4 e01 = lds_v4(st_u32 + t * 8);
                            const int4 e23 = lds_v4(st_u32 + t * 8 + 16);
                            fma_lds<VEC>(acc[r], __int_as_float(e01.y), panel + e01.x);
                            fma_lds<VEC>(acc[r], __int_as_float(e01.w), panel + e01.z);
                            fma_lds<VEC>(acc[r], __int_as_float(e23.y), panel + e23.x);
                            fma_lds<VEC>(acc[r], __int_as_float(e23.w), panel + e23.z);
                        }
                        base += cnt;
                        if (cnt < 32) break;
                        __syncwarp();
                        const int k = base + lane;  // a full warp-load was inside the panel: keep going
                        c = (k < rend) ? ld_stream(idx + k) : 0x7fffffff;
                        v = (k < rend) ? ld_stream(val + k) : 0.f;
                    }
                    if (lane == r) cur = base;
                }
            }
            ++consumed;
            __syncthreads();  // every warp is done with this buffer
            if (tid == 0 && p + 2 < n_panels) issue(p + 2);
        }
        // epilogue: 32 coalesced row stores per warp
#pragma unroll
        for (int r = 0; r < 32; ++r) {
            const int64_t row = row0 + r;
            if (row < n_rows) {
                float* dst = C + (size_t)row * P + lane * VEC;
                float o[VEC];
#pragma unroll
                for (int e = 0; e < VEC; ++e) o[e] = acc[r][e];
                if (accumulate) {
#pragma unroll
                    for (int e = 0; e < VEC; ++e) o[e] += dst[e];
                }
                if constexpr (VEC == 1) dst[0] = o[0];
                else if constexpr (VEC == 2) *reinterpret_cast<float2*>(dst) = make_float2(o[0], o[1]);
                else *reinterpret_cast<float4*>(dst) = make_float4(o[0], o[1], o[2], o[3]);
            }
        }
    }
}

template <int P>
static int launch_panel(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_rows,
                        int32_t n_cols, const float* B, float* C, int accumulate, cudaStream_t stream) {
    using Cfg = PanelCfg<P>;
    int dev = 0, max_smem = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    const int budget = max_smem - 1024 - Cfg::WARPS * 64 * 8;  // barriers, per-warp staging, slack
    int panel_cols = (budget / 2) / (P * (int)sizeof(float));
    panel_cols &= ~7;
    if (panel_cols > n_cols) panel_cols = (n_cols + 7) & ~7;
    if (panel_cols < 8) panel_cols = 8;
    const size_t smem = (size_t)2 * panel_cols * P * sizeof(float) + 64 + (size_t)Cfg::WARPS * 64 * 8;
    cudaError_t e = cudaFuncSetAttribute(spmm_csr_panel_kernel<P>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) {
        set_error("spmm_csr_panel: cudaFuncSetAttribute(%zu B smem): %s", smem, cudaGetErrorString(e));
        return -2;
    }
    const int64_t n_blocks = (n_rows + Cfg::ROWS - 1) / Cfg::ROWS;
    int grid = (int)(n_blocks < sm_count() ? n_blocks : sm_count());
    if (grid < 1) grid = 1;
    spmm_csr_panel_kernel<P><<<grid, Cfg::THREADS, smem, stream>>>(indptr, indices, data, n_rows, n_cols, B, C,
                                                                  accumulate, panel_cols);
    return check_launch("spmm_csr_panel");
}

}  // namespace mub

extern "C" int mub_spmm_csr_panel_f32(const int64_t* indptr, const int32_t* indices, const float* data,
                                      int64_t n_rows, int64_t n_cols, const float* B, int32_t ld, float* C,
                                      int32_t accumulate, mub_stream_t stream) {
    MUB_REQUIRE(n_rows >= 0 && n_cols >= 0 && n_cols < 0x7fffffff, "spmm_csr_panel: bad shape");
    MUB_REQUIRE(ld == 32 || ld == 64 || ld == 128, "spmm_csr_panel: ld must be 32, 64 or 128 (got %d)", ld);
    if (n_rows == 0) return 0;
    MUB_REQUIRE(indptr && B && C, "spmm_csr_panel: null pointer");
    MUB_REQUIRE((((uintptr_t)B | (uintptr_t)C) & 15) == 0, "spmm_csr_panel: B and C must be 16-byte aligned");
    cudaStream_t s = (cudaStream_t)stream;
    switch (ld) {
        case 32: return mub::launch_panel<32>(indptr, indices, data, n_rows, (int32_t)n_cols, B, C, accumulate, s);
        case 64: return mub::launch_panel<64>(indptr, indices, data, n_rows, (int32_t)n_cols, B, C, accumulate, s);
        default: return mub::launch_panel<128>(indptr, indices, data, n_rows, (int32_t)n_cols, B, C, accumulate, s);
    }
}
