// coach_b200/csrc/common.cuh -- shared helpers for the sm_90a kernels behind include/coach_b200.h
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/coach_b200.h"

namespace cb200 {

// ---- error plumbing (C-ABI returns int; message retrievable through cb200_last_error) ------------------------
void set_error(const char* fmt, ...);

#define CB200_CHECK_ARG(cond, msg)                                    \
    do {                                                              \
        if (!(cond)) {                                                \
            cb200::set_error("%s: %s", __func__, msg);                \
            return CB200_ERR_INVALID_ARGUMENT;                        \
        }                                                             \
    } while (0)

#define CB200_CHECK_LAUNCH()                                                              \
    do {                                                                                  \
        cudaError_t e__ = cudaGetLastError();                                             \
        if (e__ != cudaSuccess) {                                                         \
            cb200::set_error("%s: CUDA error %d (%s)", __func__, (int)e__,                \
                             cudaGetErrorString(e__));                                    \
            return CB200_ERR_CUDA;                                                        \
        }                                                                                 \
    } while (0)

#define CB200_CUDA(call)                                                                  \
    do {                                                                                  \
        cudaError_t e__ = (call);                                                         \
        if (e__ != cudaSuccess) {                                                         \
            cb200::set_error("%s: %s -> CUDA error %d (%s)", __func__, #call, (int)e__,   \
                             cudaGetErrorString(e__));                                    \
            return CB200_ERR_CUDA;                                                        \
        }                                                                                 \
    } while (0)

static inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

// what cb200_last_dispatch() reports: the kernel the calling thread's last GEMM call launched (a static string), the
// A^T fetch mode of a weight-gradient call (or NULL) and the split-reduction kernel (reset by set_dispatch)
void set_dispatch(const char* kernel, const char* fetch = nullptr);
void set_dispatch_reduce(const char* reduce);

int sm_count();   // cached multiprocessor count of the current device
// per-device caches (function attributes such as a dynamic shared memory opt-in are set per device) are indexed by the
// device ordinal
constexpr int kMaxDevices = 64;
int tune_get(const char* key, int dflt, int lo, int hi);   // runtime knob set through cb200_tune()

// ---- PTX wrappers: mbarrier + bulk async copies (TMA, 1-D form; SASS: UBLKCP / SYNCS) ---------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE;\n"
        "bra WAIT_LOOP;\n"
        "DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// global -> shared, completion signalled on an mbarrier (complete_tx)
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(smem_dst)),
        "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
// shared -> global, tracked by the per-thread bulk async-group
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst),
                 "r"(smem_u32(smem_src)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait_all() {
    asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// 16-byte streaming load/store (used by the LSU fall-back paths)
__device__ __forceinline__ int4 ld_stream16(const void* p) {
    int4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}
__device__ __forceinline__ void st_stream16(void* p, const int4& v) {
    asm volatile("st.global.L1::no_allocate.v4.s32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
                 "r"(v.w)
                 : "memory");
}

}  // namespace cb200

// ---- launch accounting ------------------------------------------------------------------------------------------
namespace cb200 {
void count_launch(int n = 1);
}
#define CB200_LAUNCH(kernel, grid, block, smem, stream, ...)        \
    do {                                                            \
        kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__); \
        cb200::count_launch();                                      \
    } while (0)
