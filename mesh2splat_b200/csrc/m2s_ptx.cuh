// m2s_ptx.cuh — the PTX the conversion kernels use directly: mbarrier + 1-D bulk async copy (TMA engine; SASS UBLKCP),
// system-scope release / acquire, the early trigger of programmatic dependent launch, and the bounded wait of the fused
// gather; and the warp scan of the kernels' and the viewer's prefix sums.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace m2s {

// inclusive prefix sum of v over the lanes of each `width`-lane segment of the warp (width: a power of two <= 32)
template <typename T>
__device__ __forceinline__ T warp_inclusive_scan(T v, int lane, int width = 32) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const T y = __shfl_up_sync(0xffffffffu, v, d, width);
        if ((lane & (width - 1)) >= d) v += y;
    }
    return v;
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void tma_load_1d(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void tma_store_1d(void* dst_gmem, const void* src_smem, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem), "r"(smem_u32(src_smem)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// the bulk groups of this thread but the most recent one have finished reading their sources
__device__ __forceinline__ void tma_store_wait_read_but_last() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// 8 bytes global -> shared without a register round trip (LDGSTS): the copy flies while the thread goes on
__device__ __forceinline__ void cp_async_8(void* dst_smem, const void* src_gmem) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(dst_smem)), "l"(src_gmem) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
// programmatic dependent launch: the grid launched behind this one may be scheduled once every CTA of this grid has
// executed this or exited.  Its griddepcontrol.wait still waits for this grid to complete and its memory to be flushed
__device__ __forceinline__ unsigned long long atom_add_acq_rel_gpu(unsigned long long* p, unsigned long long v) {
    unsigned long long old;
    asm volatile("atom.add.acq_rel.gpu.global.u64 %0, [%1], %2;" : "=l"(old) : "l"(p), "l"(v) : "memory");
    return old;
}
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ unsigned long long gtimer_ns() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
// Bounded wait for a peer's flag (fused gather): a rank that never launches its kernels must not hang every GPU of the
// node forever.  After kSpinTimeoutNs the waiter gives up, raises bit `why` in the context's status word (mapped pinned
// host memory, read by m2s_ctx_status) and carries on with whatever it has — the host call then reports M2S_E_CUDA.
constexpr unsigned long long kSpinTimeoutNs = 2000000000ull;
__device__ __forceinline__ bool wait_epoch(const unsigned long long* flag, unsigned long long epoch, uint32_t* status, uint32_t why) {
    if (ld_acquire_sys(flag) == epoch) return true;
    const unsigned long long t0 = gtimer_ns();
    unsigned ns = 100;
    while (ld_acquire_sys(flag) != epoch) {
        __nanosleep(ns);
        ns = min(ns * 2u, 2000u);
        if (gtimer_ns() - t0 > kSpinTimeoutNs) {
            if (status) { *reinterpret_cast<volatile uint32_t*>(status) = why; __threadfence_system(); }  // plain store: zero-copy memory
            return false;
        }
    }
    return true;
}
#define SCHED(a, i) ((a).sched + (i) * kSchedStride)

}  // namespace m2s
