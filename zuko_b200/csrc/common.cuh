// zuko_b200 — shared host/device helpers (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>
#include <string>

#include "../../include/zuko_b200.h"

namespace zk {

// ---------------------------------------------------------------------------
// error plumbing
// ---------------------------------------------------------------------------
extern thread_local std::string g_last_error;
extern std::atomic<int64_t> g_launches;
extern std::atomic<int> g_fast_math;
extern std::atomic<int> g_fused;

zk_status fail(zk_status code, const char* fmt, ...);

#define ZK_CUDA(expr)                                                                   \
    do {                                                                                \
        cudaError_t _e = (expr);                                                        \
        if (_e != cudaSuccess)                                                          \
            return zk::fail(ZK_ECUDA, "%s:%d: %s -> %s", __FILE__, __LINE__, #expr,     \
                            cudaGetErrorString(_e));                                    \
    } while (0)

#define ZK_TRY(expr)                    \
    do {                                \
        zk_status _s = (expr);          \
        if (_s != ZK_OK) return _s;     \
    } while (0)

#define ZK_REQUIRE(cond, ...)                                   \
    do {                                                        \
        if (!(cond)) return zk::fail(ZK_EINVAL, __VA_ARGS__);   \
    } while (0)

inline zk_status check_launch(const char* what) {
    g_launches.fetch_add(1, std::memory_order_relaxed);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(ZK_ECUDA, "launch of %s failed: %s", what, cudaGetErrorString(e));
    return ZK_OK;
}

int sm_count();  // cached, current device

// eps of BoundedBernsteinTransform in flow layers (zk_layer_desc carries no eps)
constexpr float kBernsteinEps = 1e-6f;

// A univariate bijector and its scalars (families: uni_family.cuh)
struct UniSpec {
    int kind = ZK_UNI_RQS;      // ZK_UNI_* (circular RQS: ZK_UNI_RQS with `circular`)
    int K = 0;                  // bins (RQS) / mixture components (Gaussianization) / polynomials (SOSP)
    int degree = 0;             // SOSP: polynomial degree L; Bernstein: BPF degree (P = degree + 1)
    float bound = 5.f;          // spline bound, or the bisection interval [-bound, bound]
    float slope = 1e-3f;
    float eps = kBernsteinEps;  // Bernstein: branch threshold on t = (x + bound) / 2 bound
    int iters = 0;              // Gaussianization / SOSP / Bernstein inverse: bisection steps
    bool circular = false;      // RQS only: CircularShiftTransform(bound) in front (forward) / behind (inverse)
};

inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// ---------------------------------------------------------------------------
// device-side PTX wrappers (mbarrier, bulk async copy = TMA 1-D)
// ---------------------------------------------------------------------------
#ifdef __CUDACC__

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}

// make mbarrier.init visible to the async proxy (TMA engine)
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
                 "r"(bytes)
                 : "memory");
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return done != 0;
}

// non-blocking probe (try_wait may suspend the thread for a system-dependent time before it
// reports failure — possibly thousands of cycles — so look-ahead polls must use test_wait)
__device__ __forceinline__ bool mbar_test_wait(uint64_t* bar, uint32_t parity) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return done != 0;
}

__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}

// 1-D bulk async copy global -> shared (TMA engine, SASS UBLKCP); bytes % 16 == 0,
// both addresses 16-byte aligned.  Completion is signalled on `bar` (complete_tx).
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes,
                                         uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
            "r"(smem_u32(smem_dst)),
        "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}

__device__ __forceinline__ float ld_stream(const float* p) {
    float v;
    asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
    return v;
}

#endif  // __CUDACC__

}  // namespace zk
