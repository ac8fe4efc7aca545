// Shared device/host helpers for the zigma_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>

#include "../../include/zigma_b200.h"

// ---- host side error plumbing -----------------------------------------------------------------
int zg_set_error(const char *fmt, ...);          // returns 1
void zg_count_launch(int n = 1);
int zg_check_launch(const char *what);           // cudaPeekAtLastError -> error code
void zg_note_scan_kernel(const char *name);      // which forward-scan kernel the last zg_selective_scan_fwd launched (zg_last_scan_kernel)

#define ZG_REQUIRE(cond, ...)                        \
    do {                                             \
        if (!(cond)) return zg_set_error(__VA_ARGS__); \
    } while (0)

static inline int zg_dtype_size(int dt) { return dt == ZG_F32 ? 4 : 2; }

// ---- deterministic backward (the *_bwd_det entry points) ---------------------------------------
// The DET instantiation of a backward kernel stores each value it would have added with an fp32 atomic into its own row
// of a partials region: rows x n floats, the row fixed by the static grid mapping (tile, batch row, chunk index).
// zg_reduce_rows then adds the rows into the zero-filled output in row order, so the result does not depend on the
// order in which CTAs ran.  ZgDetLayout carves one region per reduced output out of the caller's workspace; the same
// code sizes the workspace (ws == nullptr) and hands out the region pointers, so the size query and the launch agree.
int zg_reduce_rows(const float *part, int64_t rows, int64_t n, float *out, cudaStream_t s);

struct ZgDetLayout {
    struct Region { float *out, *part; int64_t rows, n; };
    Region reg[8];
    int count = 0;
    int64_t bytes = 0;
    unsigned char *ws = nullptr;
    // region of rows x n floats for `out` (nothing when out is NULL); returns where the kernel writes its partials
    float *add(float *out, int64_t rows, int64_t n) {
        if (out == nullptr || rows <= 0 || n <= 0) return nullptr;
        float *part = ws ? reinterpret_cast<float *>(ws + bytes) : nullptr;
        reg[count++] = Region{out, part, rows, n};
        bytes += (rows * n * (int64_t)sizeof(float) + 15) / 16 * 16;
        return part;
    }
    int reduce(cudaStream_t s) const {
        for (int i = 0; i < count; ++i)
            if (int rc = zg_reduce_rows(reg[i].part, reg[i].rows, reg[i].n, reg[i].out, s)) return rc;
        return 0;
    }
};
// checks the caller's workspace against the layout (which must have been built with ws set)
#define ZG_REQUIRE_WORKSPACE(lay, ws, ws_bytes, who)                                                                  \
    ZG_REQUIRE((lay).bytes <= (ws_bytes) && ((lay).bytes == 0 || ((ws) != nullptr && (reinterpret_cast<uintptr_t>(ws) & 15) == 0)), \
               "%s: workspace of %lld bytes (16-byte aligned) needed, got %lld", who, (long long)(lay).bytes, (long long)(ws_bytes))

// ---- device helpers ---------------------------------------------------------------------------
#define ZG_LOG2E 1.4426950408889634f
#define ZG_LN2 0.6931471805599453f

template <typename T> __device__ __forceinline__ float zg_to_float(T v);
template <> __device__ __forceinline__ float zg_to_float<float>(float v) { return v; }
template <> __device__ __forceinline__ float zg_to_float<__half>(__half v) { return __half2float(v); }
template <> __device__ __forceinline__ float zg_to_float<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

template <typename T> __device__ __forceinline__ T zg_from_float(float v);
template <> __device__ __forceinline__ float zg_from_float<float>(float v) { return v; }
template <> __device__ __forceinline__ __half zg_from_float<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 zg_from_float<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

__device__ __forceinline__ float zg_ex2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float zg_lg2(float x) {
    float y;
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float zg_rcp(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// softplus with the reference's threshold (selective_scan_fwd_kernel.cuh:153-156): x <= 20 ?
// log1p(exp(x)) : x.  exp via MUFU.EX2; log1p via a series for tiny e (where lg2.approx of 1+e has
// no relative accuracy) and MUFU.LG2 otherwise.  Relative error < 2e-6 over the whole range.
__device__ __forceinline__ float zg_softplus20(float x) {
    // branch free (selects): the scan's inner loop must not pay divergence bookkeeping per step
    const float e = zg_ex2(fminf(x, 20.f) * ZG_LOG2E);
    // log1p(e) = e - e^2/2 + e^3/3 - e^4/4 + e^5/5   (|err| < e^6/6 < 2e-10 * e for e < 1/32)
    const float series = e * (1.f + e * (-0.5f + e * (0.33333334f + e * (-0.25f + e * 0.2f))));
    const float viaLog = zg_lg2(1.f + e) * ZG_LN2;
    const float sp = (e < 0.03125f) ? series : viaLog;
    return (x > 20.f) ? x : sp;
}

// softplus'(x) = sigmoid(x) = 1 - exp(-softplus(x)), from sp = softplus(x) (the value the scan already holds).  Below
// sp = 1/8 (x below about -2) the difference 1 - exp(-sp) cancels -- at x = -30 it is 0 in fp32, where sigmoid(x) = 9e-14 --
// so there it is the series sp (1 - sp/2 (1 - sp/3 (1 - sp/4 (1 - sp/5 (1 - sp/6))))), relative error < sp^6 / 5040 < 1e-9.
__device__ __forceinline__ float zg_softplus_grad(float sp) {
    const float series = sp * (1.f - 0.5f * sp * (1.f - sp * (1.f / 3.f) * (1.f - 0.25f * sp * (1.f - 0.2f * sp * (1.f - sp * (1.f / 6.f))))));
    return sp < 0.125f ? series : 1.f - zg_ex2(-sp * ZG_LOG2E);
}
__device__ __forceinline__ float zg_sigmoid(float x) { return zg_rcp(1.f + zg_ex2(-x * ZG_LOG2E)); }
__device__ __forceinline__ float zg_silu(float x) { return x * zg_sigmoid(x); }

// ---- fp32 pairs: Hopper has no packed FFMA2 / FMUL2 / FADD2, so each lane is one scalar round-to-nearest op ----
typedef float2 zg_f2;
__device__ __forceinline__ zg_f2 zg_pack2(float lo, float hi) { return make_float2(lo, hi); }
__device__ __forceinline__ zg_f2 zg_splat2(float v) { return make_float2(v, v); }
__device__ __forceinline__ zg_f2 zg_fma2(zg_f2 a, zg_f2 b, zg_f2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ zg_f2 zg_mul2(zg_f2 a, zg_f2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ zg_f2 zg_add2(zg_f2 a, zg_f2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
// 2^x for two lanes at once via MUFU.EX2 (2 MUFU issues)
__device__ __forceinline__ zg_f2 zg_ex2_mufu2(zg_f2 x) { return make_float2(zg_ex2(x.x), zg_ex2(x.y)); }

// cp.async (LDGSTS) 16-byte copy global -> shared, L2 only (streamed data, no L1 allocation)
__device__ __forceinline__ void zg_cp_async16(void *smem_dst, const void *gmem_src) {
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void zg_cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void zg_cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

__device__ __forceinline__ float zg_warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ---- mbarrier + bulk async copy (TMA engine, SASS: UBLKCP / SYNCS) -------------------------------------------
__device__ __forceinline__ uint32_t zg_smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void zg_mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(zg_smem_u32(bar)), "r"(count) : "memory");
}
// makes the initialised barriers visible to the async proxy (the TMA engine signals them)
__device__ __forceinline__ void zg_mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void zg_mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(zg_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void zg_mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "ZG_WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra ZG_WAIT_DONE;\n\t"
        "bra ZG_WAIT_LOOP;\n\t"
        "ZG_WAIT_DONE:\n\t"
        "}\n" ::"r"(zg_smem_u32(bar)), "r"(parity) : "memory");
}
// global -> shared bulk copy of `bytes` (multiple of 16; both addresses 16-byte aligned), completion counted on `bar`
__device__ __forceinline__ void zg_bulk_g2s(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(zg_smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(zg_smem_u32(bar))
                 : "memory");
}
