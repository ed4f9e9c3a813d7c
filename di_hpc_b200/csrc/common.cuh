// common.cuh -- host/device plumbing shared by every op of the trajectory-return path.
//
// sm_90a (H100) only.  No torch types: this translation unit family builds into the C-ABI library
// declared in include/hpc_rll_b200.h.
//
// Replaces (re-derived, not copied) the reference's helper headers
//   include/hpc/rll/cuda/status.h:15-28  (checkCudaErr -> std::logic_error)  -> error codes + message
//   include/hpc/rll/cuda/reduce.h:13-99  (warp/block reductions)             -> reduce.cuh
//   include/hpc/rll/cuda/common.h:44-45  (DEFAULT_WARP_NUM / WARP_SIZE)      -> per-kernel constants
#pragma once

#include <cuda.h>  // CUtensorMap + enums only; the driver entry point is fetched at run time
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdarg>
#include <cstdio>

#include <nvtx3/nvToolsExt.h>  // header-only in CUDA 12: ranges cost a few ns unless a profiler is attached

#include "../../include/hpc_rll_b200.h"

namespace hpcrll {

// ----------------------------------------------------------------------------------------------
// error reporting (thread-local message, C-ABI returns the code)
// ----------------------------------------------------------------------------------------------
int set_error(int code, const char* fmt, ...);
void clear_error();

#define HPC_REQUIRE(cond, ...)                                          \
    do {                                                                \
        if (!(cond)) return ::hpcrll::set_error(HPC_RLL_EINVAL, __VA_ARGS__); \
    } while (0)

#define HPC_CUDA(expr)                                                                            \
    do {                                                                                          \
        cudaError_t e__ = (expr);                                                                 \
        if (e__ != cudaSuccess)                                                                   \
            return ::hpcrll::set_error(HPC_RLL_ECUDA, "%s failed: %s (%s:%d)", #expr,             \
                                       cudaGetErrorString(e__), __FILE__, __LINE__);              \
    } while (0)

#define HPC_LAUNCH_CHECK() HPC_CUDA(cudaGetLastError())

inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

// one NVTX range per C-ABI entry point (SURVEY.md section 5: the reference has only TRACE/printf debugging,
// include/hpc/rll/cuda/common.h:17-20); shows up in nsys / ncu --nvtx timelines as "hpc_rll:<entry>"
struct NvtxRange {
    explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
    NvtxRange(const NvtxRange&) = delete;
    NvtxRange& operator=(const NvtxRange&) = delete;
};
#define HPC_NVTX(name) ::hpcrll::NvtxRange nvtx_range__("hpc_rll:" name)

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
inline bool aligned8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7u) == 0; }

// number of SMs of the current device (cached)
int sm_count();

// every kernel launch of the library is counted (hpc_rll_launch_count)
void count_launch(int n = 1);

// ----------------------------------------------------------------------------------------------
// TMA descriptors (host).  2-D fp32 row-major view: rows x cols, row pitch ld (elements).
// Requirements: base 16B aligned, ld*4 % 16 == 0.  OOB elements of a box read as zero.
// ----------------------------------------------------------------------------------------------
bool tma_ok_2d(const void* base, int64_t cols, int64_t ld);
int make_tmap_2d(CUtensorMap* out, const float* base, int64_t rows, int64_t cols, int64_t ld, int box_rows,
                 int box_cols, bool swizzle128 = false);  // swizzle128: CU_TENSOR_MAP_SWIZZLE_128B (box_cols <= 32)
// the same for a uint8 tensor (masks): base 16B aligned, ld % 16 == 0, box_cols % 16 == 0
int make_tmap_2d_u8(CUtensorMap* out, const uint8_t* base, int64_t rows, int64_t cols, int64_t ld, int box_rows,
                    int box_cols);

// Opt a kernel into more dynamic shared memory than it may use by default: 48 KB minus its static shared memory (a
// launch above that fails).  The first opt-in also sets the kernel's carveout to the largest shared-memory share.  The
// attribute is per context and holds the LARGEST byte count granted so far per device: kernels whose dynamic size
// varies at run time (n_atom / tau dependent, nstep.cu) are re-opted whenever a call needs more than any earlier one
// (ADVICE r1: a first call at ~50 KB used to pin the limit).
struct SmemOptIn {
    int granted[64] = {};
    template <typename K>
    int ensure(K kernel, int bytes) {
        int dev = 0;
        HPC_CUDA(cudaGetDevice(&dev));
        const bool tracked = dev >= 0 && dev < 64;
        if (tracked && granted[dev] >= bytes && granted[dev] > 0) return HPC_RLL_OK;
        HPC_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
        if (!tracked || granted[dev] == 0)
            HPC_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                                          cudaSharedmemCarveoutMaxShared));
        if (tracked) granted[dev] = bytes;
        return HPC_RLL_OK;
    }
};

// scratch requirement of each op (defined next to the op's kernels; runtime.cu dispatches)
size_t workspace_bytes(int op, int64_t T, int64_t B, int64_t N);

// debug/tuning knob: HPC_RLL_CFG_<op> environment override or hpc_rll_debug_set_config()
int tuning_config(int op);

// ----------------------------------------------------------------------------------------------
// device: mbarrier + TMA PTX wrappers
// ----------------------------------------------------------------------------------------------
#ifdef __CUDACC__

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
// make mbarrier.init visible to the async proxy (TMA) before the first copy targets it
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}

// 2-D tiled TMA load: box at (col0,row0) of the tensor map -> smem, completes on `bar`
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int col0, int row0, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(col0), "r"(row0), "r"(smem_u32(bar))
        : "memory");
}
// 1-D bulk copy global -> smem (bytes % 16 == 0, both 16B aligned), completes on `bar`
__device__ __forceinline__ void bulk_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst)),
                 "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// 2-D tiled TMA store: smem box -> (col0,row0) of the tensor map; elements outside the tensor are clipped.
// Completion is tracked by bulk async-groups of the issuing thread (commit + wait below).
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, int col0, int row0, const void* src) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%1, %2}], [%3];" ::"l"(
                     reinterpret_cast<uint64_t>(map)),
                 "r"(col0), "r"(row0), "r"(smem_u32(src))
                 : "memory");
}
// 1-D bulk copy smem -> global (bytes % 16 == 0, both 16B aligned); completion by bulk async-groups as above
__device__ __forceinline__ void bulk_store_1d(void* dst, const void* src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(reinterpret_cast<uint64_t>(dst)),
                 "r"(smem_u32(src)), "r"(bytes)
                 : "memory");
}
// same with an L2 eviction-priority hint (createpolicy): data the next kernel re-reads should stay resident
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void bulk_store_1d_hint(void* dst, const void* src, uint32_t bytes, uint64_t policy) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;" ::"l"(
                     reinterpret_cast<uint64_t>(dst)),
                 "r"(smem_u32(src)), "r"(bytes), "l"(policy)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// wait until at most N of this thread's bulk groups are still READING shared memory
template <int N>
__device__ __forceinline__ void bulk_wait_group_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
// wait until at most N of this thread's bulk groups are pending at all (writes performed)
template <int N>
__device__ __forceinline__ void bulk_wait_group() {
    asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
// named barrier over `count` threads (a multiple of 32) of the CTA; id 0 is __syncthreads
__device__ __forceinline__ void named_bar_sync(int id, int count) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

// streaming (evict-first) global accesses for data touched exactly once
__device__ __forceinline__ void st_stream(float* p, float v) { __stcs(p, v); }
__device__ __forceinline__ void st_stream2(float2* p, float2 v) { __stcs(p, v); }
__device__ __forceinline__ void st_stream4(float4* p, float4 v) { __stcs(p, v); }
__device__ __forceinline__ float ld_stream(const float* p) { return __ldcs(p); }
__device__ __forceinline__ float4 ld_stream4(const float4* p) { return __ldcs(p); }
// one byte of a mask tensor; a NULL mask reads as 0 (not set)
__device__ __forceinline__ unsigned ld_mask(const uint8_t* __restrict__ p, int64_t i) {
    return p != nullptr ? static_cast<unsigned>(__ldg(reinterpret_cast<const unsigned char*>(p) + i)) : 0u;
}

#endif  // __CUDACC__

}  // namespace hpcrll
