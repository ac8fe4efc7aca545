// bf16 GEMM on the Hopper tensor cores (wgmma + TMA + mbarrier + thread-block clusters), hand written for sm_90a.
//
//     C[M, N] = A[M, K] * B[N, K]^T (+ bias[N])        A, B, C row-major bf16, fp32 accumulation in registers
//
// This is the shape of every dense projection on the ZigMa hot path in the token-major layout (DESIGN.md
// section 3): in_proj (mamba_simple.py:290-294), x_proj / dt_proj (selective_scan_interface.py:322-323)
// and out_proj (:365) -- activations (B*L, K) times an nn.Linear weight (N, K).  The reference leaves them
// to cuBLAS behind F.linear / `@`.
//
// Structure (one CTA per SM, persistent over output tiles; 384 threads = three warpgroups):
//   warpgroup 0   TMA producer (registers handed back with setmaxnreg): one lane issues cp.async.bulk.tensor loads
//            of the A (128 x 64) and B (BN x 64) k-blocks into a shared-memory ring (128-byte swizzle), mbarrier
//            tx-count.
//   warpgroups 1-2   consumers: each owns 64 of the tile's 128 rows and issues wgmma.mma_async m64 x BN x k16 (both
//            operands from shared memory, K-major), 4 per k-block, keeping one k-block in flight; a stage goes back
//            to the producer once the wgmmas that read it have retired.  Epilogue from the accumulator fragments:
//            (+bias) -> bf16 -> swizzled shared memory -> TMA store (16 rows x 64 columns per warp, asynchronous, so
//            it drains under the next tile's main loop), or direct stores through `out_rowmap` (row scatter of the
//            out_proj result back to raster order, mamba_simple.py:388-394).
// K, M, N remainders are handled by TMA out-of-bounds zero fill (loads) and clipped / predicated stores.
//
// Thread-block clusters (CL = 2 or 4 CTAs along M): every 128 x BN output tile re-reads its BN x K weight tile from
// L2.  The CTAs of a cluster work on CL vertically adjacent output tiles that share the weight tile; each CTA fetches
// 1/CL of it and TMA-multicasts the slice into the shared memory of all CL CTAs.  A stage may only be overwritten once
// EVERY CTA of the cluster has consumed it: each consumer warp arrives on the `empty` barrier of all CTAs of the
// cluster (remote mbarrier arrive), whose arrival count is 8 warps x CL.
#include "zg_common.cuh"
#include <cuda.h>
#include <stdlib.h>

namespace zg {

constexpr int G_BM = 128, G_BK = 64, G_THREADS = 384;   // 3 warpgroups: TMA producer, 2 consumers of 64 rows each
constexpr int G_EPI_BYTES = 8 * 2 * 16 * 128;           // per consumer warp two (16 rows x 128 B) swizzled buffers for the TMA store
// smem ring depth: as many (128 + BN) x 64 bf16 stages as fit next to the epilogue staging
__host__ __device__ constexpr int gemm_stages(int BN) {
    const int stage = (G_BM + BN) * G_BK * 2, avail = 227 * 1024 - G_EPI_BYTES - 2048;
    return avail / stage > 8 ? 8 : avail / stage;
}

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra WAIT_DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "WAIT_DONE:\n\t"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void *dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
                 "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void tma_load_2d_mc(void *dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1, uint16_t mask) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(
                     smem_u32(dst)),
                 "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(mask)
                 : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
// arrive on the barrier at this shared-memory offset in CTA `cta` of the cluster
__device__ __forceinline__ void mbar_arrive_remote(uint64_t *bar, uint32_t cta) {
    uint32_t ra;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(smem_u32(bar)), "r"(cta));
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(ra) : "memory");
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared-memory matrix descriptor of a wgmma operand: K-major, 128-byte swizzle, rows of 64 bf16 (128 B), 8-row groups
// 1024 B apart (PTX ISA "Matrix Descriptor Format": start >> 4 at [0,14), leading byte offset >> 4 at [16,30) -- unused for
// swizzled K-major, canonical value 1 --, stride byte offset >> 4 at [32,46), swizzle mode at [62,64): 1 = 128 bytes).
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3ffff) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator registers across an asynchronous wgmma that still writes them
template <int R> __device__ __forceinline__ void fence_accumulators(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, one warpgroup, both operands through shared-memory descriptors; `accumulate` == 0
// overwrites D.  Thread t of the warpgroup holds rows (t / 32) * 16 + (t % 32) / 4 (+ 8) and, for each group j of 8 columns,
// columns 8 j + 2 (t % 4) (+ 1): d[4 j + 0 .. 1] for the first row, d[4 j + 2 .. 3] for the row 8 below.
template <int N> struct Wgmma;
template <> struct Wgmma<64> {
    static __device__ __forceinline__ void mma(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
        asm volatile(
            "{\n\t"
            ".reg .pred p;\n\t"
            "setp.ne.b32 p, %34, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
            "%32, %33, p, 1, 1, 0, 0;\n\t"
            "}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "l"(adesc), "l"(bdesc), "r"(accumulate));
    }
};

template <> struct Wgmma<80> {
    static __device__ __forceinline__ void mma(float (&d)[40], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
        asm volatile(
            "{\n\t"
            ".reg .pred p;\n\t"
            "setp.ne.b32 p, %42, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n80k16.f32.bf16.bf16 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
            "%32, %33, %34, %35, %36, %37, %38, %39}, "
            "%40, %41, p, 1, 1, 0, 0;\n\t"
            "}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
              "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
            : "l"(adesc), "l"(bdesc), "r"(accumulate));
    }
};

template <> struct Wgmma<128> {
    static __device__ __forceinline__ void mma(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
        asm volatile(
            "{\n\t"
            ".reg .pred p;\n\t"
            "setp.ne.b32 p, %66, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
            "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
            "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
            "%64, %65, p, 1, 1, 0, 0;\n\t"
            "}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
              "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
              "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
              "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
              "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
            : "l"(adesc), "l"(bdesc), "r"(accumulate));
    }
};

template <> struct Wgmma<160> {
    static __device__ __forceinline__ void mma(float (&d)[80], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
        asm volatile(
            "{\n\t"
            ".reg .pred p;\n\t"
            "setp.ne.b32 p, %82, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n160k16.f32.bf16.bf16 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
            "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
            "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
            "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79}, "
            "%80, %81, p, 1, 1, 0, 0;\n\t"
            "}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
              "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
              "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
              "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
              "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
              "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
              "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79])
            : "l"(adesc), "l"(bdesc), "r"(accumulate));
    }
};

template <> struct Wgmma<256> {
    static __device__ __forceinline__ void mma(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
        asm volatile(
            "{\n\t"
            ".reg .pred p;\n\t"
            "setp.ne.b32 p, %130, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
            "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
            "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
            "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
            "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
            "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
            "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
            "%128, %129, p, 1, 1, 0, 0;\n\t"
            "}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
              "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
              "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
              "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
              "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
              "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
              "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
              "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
              "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
              "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
              "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
              "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
              "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
            : "l"(adesc), "l"(bdesc), "r"(accumulate));
    }
};

struct GemmArgs {
    __nv_bfloat16 *C;
    const __nv_bfloat16 *bias;
    const int32_t *out_rowmap;
    int64_t ldc;
    int M, N, K, rows_per_batch;
    int tma_store;      // 1: epilogue goes through smem + TMA store (needs 16-byte aligned C rows)
};

template <int BN, int CL>
__global__ void __launch_bounds__(G_THREADS, 1)
gemm_bf16_tn_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                    const __grid_constant__ CUtensorMap tmC, const GemmArgs g) {
    constexpr int BM = G_BM, BK = G_BK, STAGES = gemm_stages(BN);
    constexpr uint32_t A_BYTES = BM * BK * 2, B_BYTES = BN * BK * 2, STAGE_BYTES = A_BYTES + B_BYTES;
    extern __shared__ __align__(1024) unsigned char gsm[];
    unsigned char *tiles = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(gsm) + 1023) & ~(uintptr_t)1023);
    unsigned char *epi = tiles + STAGES * STAGE_BYTES;
    uint64_t *full_bar = reinterpret_cast<uint64_t *>(epi + G_EPI_BYTES);   // [STAGES] k-block landed (TMA tx bytes)
    uint64_t *empty_bar = full_bar + STAGES;                                // [STAGES] stage consumed by every consumer warp of the cluster

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
    const uint32_t rank = (CL > 1) ? cluster_ctarank() : 0u;
    const int cluster_id = blockIdx.x / CL, num_clusters = gridDim.x / CL;
    const int m_tiles = (g.M + BM - 1) / BM, n_tiles = (g.N + BN - 1) / BN;
    const int sm_tiles = (m_tiles + CL - 1) / CL;             // super tiles of CL vertically adjacent output tiles
    const int num_tiles = sm_tiles * n_tiles;                 // per cluster work list (identical for all its CTAs)
    const int k_blocks = (g.K + BK - 1) / BK;

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
        for (int i = 0; i < STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 8 * CL); }
        zg_mbar_fence_init();
    }
    __syncthreads();
    if (CL > 1) cluster_sync_all();          // every CTA's barriers are initialised before any remote arrive / multicast

    if (wg == 0) {
        // ===== TMA producer =====
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp == 0 && lane == 0) {
            uint32_t it = 0;
            for (int tile = cluster_id; tile < num_tiles; tile += num_clusters) {
                const int m_blk = (tile / n_tiles) * CL + (int)rank, n_blk = tile % n_tiles;
                for (int kb = 0; kb < k_blocks; ++kb, ++it) {
                    const int st = it % STAGES;
                    const uint32_t ph = (it / STAGES) & 1;
                    mbar_wait(&empty_bar[st], ph ^ 1);
                    unsigned char *sa = tiles + st * STAGE_BYTES;
                    mbar_expect_tx(&full_bar[st], STAGE_BYTES);
                    tma_load_2d(sa, &tmA, &full_bar[st], kb * BK, m_blk * BM);
                    if (CL > 1) {   // my 1/CL slice of the weight tile, multicast to the whole cluster
                        constexpr int SL = BN / CL;
                        tma_load_2d_mc(sa + A_BYTES + rank * (SL * BK * 2), &tmB, &full_bar[st], kb * BK, n_blk * BN + (int)rank * SL,
                                       (uint16_t)((1u << CL) - 1));
                    } else {
                        tma_load_2d(sa + A_BYTES, &tmB, &full_bar[st], kb * BK, n_blk * BN);
                    }
                }
            }
        }
    } else {
        // ===== consumer warpgroups 1, 2: rows [64 (wg - 1), + 64) of the tile; warp w of the warpgroup owns 16 of them =====
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        const int cw = wg - 1, q = lane & 3;
        const int wrow_in_tile = cw * 64 + (warp & 3) * 16;
        // the stage goes back to the producer of every CTA of the cluster (they all multicast into it)
        auto release = [&](int st) {
            if (lane == 0) {
                if (CL > 1) {
                    for (uint32_t c = 0; c < (uint32_t)CL; ++c) mbar_arrive_remote(&empty_bar[st], c);
                } else {
                    mbar_arrive(&empty_bar[st]);
                }
            }
        };
        unsigned char *ebuf = epi + (warp - 4) * (2 * 16 * 128);
        float d[BN / 2];
        uint32_t it = 0;
        for (int tile = cluster_id; tile < num_tiles; tile += num_clusters) {
            const int m_blk = (tile / n_tiles) * CL + (int)rank, n_blk = tile % n_tiles;
            int prev_st = 0;
            for (int kb = 0; kb < k_blocks; ++kb, ++it) {
                const int st = it % STAGES;
                const uint32_t ph = (it / STAGES) & 1;
                mbar_wait(&full_bar[st], ph);
                const uint32_t sa = smem_u32(tiles + st * STAGE_BYTES);
                const uint64_t adesc = make_smem_desc(sa + cw * (64 * BK * 2)), bdesc = make_smem_desc(sa + A_BYTES);
                fence_accumulators(d);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / 16; ++k)      // +32 B per K=16 step inside the 128-byte swizzle atom
                    Wgmma<BN>::mma(d, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), (kb | k) ? 1u : 0u);
                wgmma_commit();
                if (kb > 0) {                           // the previous k-block's wgmmas have retired: its stage is free
                    wgmma_wait<1>();
                    release(prev_st);
                }
                prev_st = st;
            }
            wgmma_wait<0>();
            fence_accumulators(d);
            release(prev_st);

            // ---- epilogue: this thread's two rows, columns 8 j + 2 q (+ 1) of every 8-column group j ----
            const int wrow = m_blk * BM + wrow_in_tile;
            const int col_lim = min(g.N, (n_blk + 1) * BN);   // first column that is NOT this tile's
            __nv_bfloat16 *crow[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = wrow + (lane >> 2) + 8 * h;
                crow[h] = nullptr;
                if (row < g.M) {
                    int64_t drow = row;
                    if (g.out_rowmap) {
                        const int bidx = row / g.rows_per_batch;
                        drow = (int64_t)bidx * g.rows_per_batch + g.out_rowmap[row - bidx * g.rows_per_batch];
                    }
                    crow[h] = g.C + drow * g.ldc;
                }
            }
            // direct store of column group j (bounds: the matrix and the tile)
            auto direct_store8 = [&](int j) {
                const int c = n_blk * BN + j * 8 + 2 * q;
                if (c >= col_lim) return;
                float b0 = 0.f, b1 = 0.f;
                if (g.bias) {
                    b0 = __bfloat162float(g.bias[c]);
                    if (c + 1 < col_lim) b1 = __bfloat162float(g.bias[c + 1]);
                }
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    if (!crow[h]) continue;
                    const float a = d[4 * j + 2 * h] + b0, b2 = d[4 * j + 2 * h + 1] + b1;
                    if (c + 1 < col_lim && ((reinterpret_cast<uintptr_t>(crow[h] + c) & 3) == 0)) {
                        *reinterpret_cast<__nv_bfloat162 *>(crow[h] + c) = __floats2bfloat162_rn(a, b2);
                    } else {
                        crow[h][c] = __float2bfloat16_rn(a);
                        if (c + 1 < col_lim) crow[h][c + 1] = __float2bfloat16_rn(b2);
                    }
                }
            };
            constexpr int NFULL = BN / 64;                    // 64-column chunks that go through the TMA store
            if (g.tma_store) {
                // ---- coalesced path: fragments -> bf16 -> swizzled smem -> TMA store (clips M/N edges) ----
#pragma unroll
                for (int ch = 0; ch < NFULL; ++ch) {
                    const int col0 = n_blk * BN + ch * 64;
                    unsigned char *buf = ebuf + (ch & 1) * (16 * 128);
                    // Every chunk commits one bulk group, also an empty one when it lies outside the matrix, so the groups alternate
                    // between the two buffers without exception: with at most one group still reading, it is the OTHER buffer's, and
                    // the store that last read this buffer (two groups ago) has finished with it.
                    if (lane == 0) {
                        if (NFULL % 2 == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
                        else asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");     // one chunk per tile: same buffer every time
                    }
                    __syncwarp();
                    if (col0 < g.N) {                          // (else: whole chunk outside the matrix)
#pragma unroll
                        for (int jj = 0; jj < 8; ++jj) {
                            const int j = ch * 8 + jj, c = col0 + jj * 8 + 2 * q;
                            float b0 = 0.f, b1 = 0.f;
                            if (g.bias) {
                                if (c < g.N) b0 = __bfloat162float(g.bias[c]);
                                if (c + 1 < g.N) b1 = __bfloat162float(g.bias[c + 1]);
                            }
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
                                // row r of the buffer, 16-byte chunk index jj XOR (r % 8): the 128-byte swizzle the TMA expects
                                const int r = (lane >> 2) + 8 * h;
                                __nv_bfloat162 v = __floats2bfloat162_rn(d[4 * j + 2 * h] + b0, d[4 * j + 2 * h + 1] + b1);
                                *reinterpret_cast<__nv_bfloat162 *>(buf + r * 128 + ((jj ^ (r & 7)) * 16) + q * 4) = v;
                            }
                        }
                        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic-proxy writes -> async proxy
                        __syncwarp();
                        if (lane == 0 && wrow < g.M)
                            asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(&tmC),
                                         "r"(smem_u32(buf)), "r"(col0), "r"(wrow)
                                         : "memory");
                    }
                    if (lane == 0) asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                }
                // tile widths that are not a multiple of 64 (80, 160): the last 16 / 32 columns leave by direct stores
#pragma unroll
                for (int j = NFULL * 8; j < BN / 8; ++j) direct_store8(j);
            } else {
                // ---- direct path (row scatter through out_rowmap, or unaligned C): 4-byte stores, 16 B per row and group ----
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) direct_store8(j);
            }
        }
        if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // my TMA stores have landed
    }
    __syncthreads();
    if (CL > 1) cluster_sync_all();          // no CTA leaves while a peer may still multicast into it / arrive on its barriers
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

// 2-D row-major bf16 matrix (rows x cols, leading dimension ld elements) -> tensor map with a (box_rows x 64) box
static int make_map(CUtensorMap *m, const void *base, int64_t rows, int64_t cols, int64_t ld, int box_rows, bool l2_promote = true) {
    EncodeTiledFn enc = get_encode();
    if (!enc) return zg_set_error("gemm_bf16_tn: cuTensorMapEncodeTiled not available from the driver");
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
    cuuint32_t box[2] = {(cuuint32_t)G_BK, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, l2_promote ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B : CU_TENSOR_MAP_L2_PROMOTION_NONE,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return zg_set_error("gemm_bf16_tn: cuTensorMapEncodeTiled failed (%d)", (int)r);
    return 0;
}

template <int BN, int CL> static int launch_gemm(const zg_gemm_params &p, cudaStream_t s) {
    CUtensorMap tmA, tmB, tmC;
    if (int rc = make_map(&tmA, p.A, p.M, p.K, p.lda, G_BM)) return rc;
    if (int rc = make_map(&tmB, p.B, p.N, p.K, p.ldb, BN / CL)) return rc;
    const bool tma_store_ok = !p.out_rowmap && p.ldc % 8 == 0 && (reinterpret_cast<uintptr_t>(p.C) & 15) == 0;
    if (tma_store_ok) {
        if (int rc = make_map(&tmC, p.C, p.M, p.N, p.ldc, 16, false)) return rc;
    } else {
        tmC = tmA;     // unused by the direct-store epilogue
    }
    GemmArgs g{reinterpret_cast<__nv_bfloat16 *>(p.C), reinterpret_cast<const __nv_bfloat16 *>(p.bias), p.out_rowmap, p.ldc, p.M, p.N, p.K,
               p.rows_per_batch > 0 ? p.rows_per_batch : p.M, tma_store_ok ? 1 : 0};
    const int smem = gemm_stages(BN) * (G_BM + BN) * G_BK * 2 + G_EPI_BYTES + 1024 + 512;
    auto kern = gemm_bf16_tn_kernel<BN, CL>;
    cudaLaunchConfig_t cfg = {};
    cfg.blockDim = dim3(G_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = CL;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    // per DEVICE (function attributes and SM counts are device state; one process may drive several GPUs)
    static int clusters_dev[64] = {};      // clusters of CL CTAs that can be resident at once (0: not asked yet)
    int dev = 0;
    cudaGetDevice(&dev);
    const int di = dev & 63;
    if (!clusters_dev[di]) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) return zg_set_error("gemm_bf16_tn: cudaFuncSetAttribute(%d): %s", smem, cudaGetErrorString(e));
        int sms = 0, n = 0;
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        cfg.gridDim = dim3(sms / CL * CL);
        // (not every GPC holds a whole number of clusters: fewer than sms / CL of them may fit)
        e = cudaOccupancyMaxActiveClusters(&n, kern, &cfg);
        if (e != cudaSuccess || n < 1) return zg_set_error("gemm_bf16_tn: no cluster of %d CTAs fits on the device: %s", CL, cudaGetErrorString(e));
        clusters_dev[di] = n < sms / CL ? n : sms / CL;
    }
    const int m_tiles = (p.M + G_BM - 1) / G_BM, n_tiles = (p.N + BN - 1) / BN;
    const int work = ((m_tiles + CL - 1) / CL) * n_tiles;          // cluster work items
    const int clusters = work < clusters_dev[di] ? work : clusters_dev[di];
    cfg.gridDim = dim3(clusters * CL);
    cudaError_t e = cudaLaunchKernelEx(&cfg, kern, tmA, tmB, tmC, g);
    zg_count_launch();
    if (e != cudaSuccess) return zg_set_error("gemm_bf16_tn: launch failed: %s", cudaGetErrorString(e));
    return zg_check_launch("gemm_bf16_tn");
}

// cluster size: ZG_GEMM_CLUSTER = 1 | 2 | 4 (default 2 when the problem has at least that many row tiles)
static int gemm_cluster_setting() {
    static int v = -1;
    if (v < 0) {
        const char *e = getenv("ZG_GEMM_CLUSTER");
        v = e ? atoi(e) : 2;
        if (v != 1 && v != 2 && v != 4) v = 2;
    }
    return v;
}

template <int BN> static int launch_gemm_cl(const zg_gemm_params &p, cudaStream_t s) {
    int cl = gemm_cluster_setting();
    const int m_tiles = (p.M + G_BM - 1) / G_BM;
    while (cl > 1 && (m_tiles < cl || (BN / cl) % 8 != 0)) cl >>= 1;     // (a CTA's multicast slice must be whole 8-row swizzle groups)
    if (cl == 4) return launch_gemm<BN, 4>(p, s);
    if (cl == 2) return launch_gemm<BN, 2>(p, s);
    return launch_gemm<BN, 1>(p, s);
}

}  // namespace zg

extern "C" int zg_gemm_bf16_tn(const zg_gemm_params *pp, void *stream) {
    ZG_REQUIRE(pp != nullptr, "gemm_bf16_tn: null params");
    const zg_gemm_params &p = *pp;
    ZG_REQUIRE(p.A && p.B && p.C, "gemm_bf16_tn: null tensor pointer");
    ZG_REQUIRE(p.M > 0 && p.N > 0 && p.K > 0, "gemm_bf16_tn: bad shape (%d, %d, %d)", p.M, p.N, p.K);
    ZG_REQUIRE(p.lda % 8 == 0 && p.ldb % 8 == 0 && p.lda >= p.K && p.ldb >= p.K && p.ldc >= p.N, "gemm_bf16_tn: leading dimensions must be multiples of 8 elements");
    ZG_REQUIRE((reinterpret_cast<uintptr_t>(p.A) & 15) == 0 && (reinterpret_cast<uintptr_t>(p.B) & 15) == 0, "gemm_bf16_tn: A and B must be 16-byte aligned");
    ZG_REQUIRE(!p.out_rowmap || (p.rows_per_batch > 0 && p.M % p.rows_per_batch == 0), "gemm_bf16_tn: out_rowmap needs rows_per_batch dividing M");
    cudaStream_t s = (cudaStream_t)stream;
    // tile width: among {256, 160, 128, 80, 64} the WIDEST whose ragged last column tile wastes <= 5 % of the MMA work, else the
    // one that wastes least (wider tiles move fewer operand bytes per MAC through L2 and re-read A fewer times).  160 exists for
    // N = 640 (out_proj of the D = 640 models: 4 x 160 exactly; 256-wide tiles pad it to 768 = 17 % idle MMAs), 80 for the
    // x_proj widths 72 / 80 (one pass over A instead of two 64-wide ones).
    static int bn_env = -1;
    if (bn_env < 0) { const char *e = getenv("ZG_GEMM_BN"); bn_env = e ? atoi(e) : 0; }
    int bn = bn_env;
    if (bn != 64 && bn != 80 && bn != 128 && bn != 160 && bn != 256) {
        const int cand[5] = {256, 160, 128, 80, 64};
        auto waste = [&](int b) { return (double)(((p.N + b - 1) / b) * b - p.N) / (double)(((p.N + b - 1) / b) * b); };
        bn = 0;
        for (int i = 0; i < 5 && !bn; ++i)
            if (waste(cand[i]) <= 0.05) bn = cand[i];
        if (!bn) {
            bn = 64;
            for (int i = 0; i < 5; ++i)
                if (waste(cand[i]) < waste(bn) - 1e-9) bn = cand[i];
        }
    }
    if (bn == 256) return zg::launch_gemm_cl<256>(p, s);
    if (bn == 160) return zg::launch_gemm_cl<160>(p, s);
    if (bn == 128) return zg::launch_gemm_cl<128>(p, s);
    if (bn == 80) return zg::launch_gemm_cl<80>(p, s);
    return zg::launch_gemm_cl<64>(p, s);
}
