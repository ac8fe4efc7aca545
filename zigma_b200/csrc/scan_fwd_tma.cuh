// Selective-scan forward, round-2 hot path: TMA-staged tiles + mbarrier pipeline, three-phase stages,
// optional fused dt_proj prologue on the tensor cores.
//
// Shape class: token-major (dim-contiguous) 16-bit activations, N = 16 states, input-dependent B/C, seqlen % 8 == 0,
// 64-channel tiles -- every ZigMa sampling / training configuration.  Semantics: selective_scan_fwd_kernel.cuh:153-171
// (delta bias + softplus), :216-261 (the recurrence h = exp(delta A) h + delta u B, y = C h), :280-298 (D skip, SiLU(z)
// gate) and, for the fused prologue, selective_scan_interface.py:323 (delta = dt_proj.weight @ x_dbl[:, :R].t()).
//
// Why a rewrite (profile of scan_fwd_tpc2_kernel on the GPU it was first tuned on): 141 issued instructions per
// (b, e, l) against 48 of state arithmetic and 20 MUFU; issue 59 %, XU 67 %.  The per-step scalar work (softplus, SiLU,
// bf16 unpacking, two SHFLs, per-thread LDGSTS address arithmetic, 2-byte stores) sat inside the recurrence loop of every
// thread, and three block barriers per 16 steps kept the four warps of a CTA in lock step.  Here:
//
//   staging    a stage = 8 steps x 64 channels.  The dense tensors (u, delta or the x_dbl rows, z when it is not gathered)
//              arrive as ONE TMA tensor tile each (cp.async.bulk.tensor.3d, SASS UTMALDG, 128-byte swizzle so that both
//              the row-wise and the MMA-fragment readers are bank-conflict free), the z rows gathered through `z_rowmap`
//              (the zigzag table) and the unfused B/C rows as 16-byte cp.async chunks; everything is counted on one
//              mbarrier per ring slot.  [A first version issued one `cp.async.bulk` (UBLKCP) per row from 32 lanes: UBLKCP
//              takes uniform registers, ptxas serialises the lanes in a waterfall loop of ~8 instructions per copy, and the
//              producer warp needed 2x the instructions of a compute warp -- 0.60 ms, slower than round 1.]
//   phases     the 128 threads of a CTA run a stage in three phases, each with the thread mapping that suits it, two
//              __syncthreads per stage (after main; after post + pre of the next stage).  [A warp-autonomous variant --
//              every warp walking the stages on its own, the last warp to release a ring slot refilling it -- was
//              measured SLOWER (0.577 vs 0.508 ms): with a 2-3 deep ring the fast warps only run ahead until they
//              block on a refill that is gated by the slowest warp, and then wait for the slowest warp AND the TMA latency.]
//   pre        delta' = softplus(delta + bias) and delta' u ONCE per (channel, step), packed fp32x2 arithmetic, written as
//              fp32 (delta', delta' u) pairs; B/C rows -> fp32.  Fused variant: the delta tile of the stage is
//              a tensor-core product (ldmatrix + mma.sync m16n8k16 / m16n8k8) of the x_dbl rows already staged for B/C with
//              the CTA's dt_proj rows (kept in shared memory), rounded to the I/O dtype like the reference's GEMM output:
//              the (batch, dim, seqlen) delta tensor never exists in HBM and the dt_proj GEMM launch disappears.
//   main       two threads per channel, 8 states (4 fp32x2 pairs) each: per step one LDS.64 (delta', delta' u), four
//              LDS.128 (B, C), 4 x {pair multiply, 2 MUFU.EX2 | polynomial, pair multiply, 2 pair FMAs}, one FADD, one STS (the partial
//              y overwrites the (delta', delta' u) slot it came from).
//   post       y = y_lo + y_hi + D u, SiLU(z) gate, bf16x2 pack, 4-byte stores.
#pragma once
#include "scan_fwd.cuh"
#include <cuda.h>
#include <string.h>
#include <type_traits>

#ifndef ZG_SCAN_EXP
#define ZG_SCAN_EXP 0      // 1, 2: timing experiments (wrong results), see DESIGN.md
#endif
#ifndef ZG_SCAN_SWP
#define ZG_SCAN_SWP 1      // hand software-pipelined recurrence loop (0: the straight loop)
#endif
#ifndef ZG_SCAN_WP_DEFAULT
#define ZG_SCAN_WP_DEFAULT -1  // -1: chosen per call (scan_auto_choice); 0: CTA-wide phases (this file); 1 / 2: warp-private pipeline (scan_fwd_wp.cuh), cp.async / TMA staging; 3 / 4: two channels per lane (scan_fwd_wp2.cuh); 5: mixed CTAs (scan_fwd_wph.cuh)
#endif
#ifndef ZG_SCAN_TMA_NPOLY_DEFAULT
#define ZG_SCAN_TMA_NPOLY_DEFAULT 0
#endif

namespace zg {

constexpr int PT_TL = 8;              // steps per stage
constexpr int PT_CH = 64;             // channels per CTA
constexpr int PT_F32ROW = 576;        // pitch of one step of the fp32 pair tile (64 channels x 8 B + 64: bank shift of 16 words)

__host__ __device__ constexpr int pt_pitch16(int bytes) { return ((bytes / 16) | 1) * 16; }   // odd number of 16-byte units

template <int R, int TPC = 2> struct PtLayout {           // R = dt_rank of the fused prologue, 0 = delta comes from HBM; TPC = threads per channel
    static constexpr bool FUSE = R > 0;
    static constexpr int NSTAGE = 3;
    static constexpr int NSWZ = FUSE ? 2 : 3;                         // swizzled 8 x 128 B tiles per stage: u, z (, delta)
    static constexpr int XBYTES = (R + 32) * 2;                       // one x_dbl row: dt | B | C (dense, unswizzled)
    static constexpr int WROW = FUSE ? pt_pitch16(2 * R) : 0;
    // 1024-byte tiles first (the 128-byte swizzle needs 1024-byte alignment), then the odd-sized ones
    static constexpr int TILE = PT_TL * 128;
    static constexpr int SWZ_OFF = 0;                                 // [stage][u, z, (delta)]
    static constexpr int X_OFF = NSTAGE * NSWZ * TILE;                // fused: x_dbl rows; unfused: raw B|C rows (64 B each)
    static constexpr int XSTAGE = FUSE ? ((PT_TL * XBYTES + 127) / 128) * 128 : PT_TL * 64;
    static constexpr int DDU_OFF = X_OFF + NSTAGE * XSTAGE;           // (delta', delta' u) fp32 pairs; the partial y overwrite them
    static constexpr int BCF_OFF = DDU_OFF + PT_TL * PT_F32ROW;       // fp32 [step][B0..15 C0..15]
    static constexpr int YROW = 64 * 4 * TPC + 64;                    // TPC > 2: separate partial-y tile, TPC floats per channel and step
    static constexpr int Y_OFF = BCF_OFF + PT_TL * 32 * 4;
    static constexpr int W_OFF = Y_OFF + (TPC > 2 ? PT_TL * YROW : 0);
    static constexpr int BAR_OFF = W_OFF + (FUSE ? PT_CH * WROW : 0);
    static constexpr int TOTAL = BAR_OFF + NSTAGE * 8;
};

// 2^x for x <= 0 (two lanes) on the FMA / ALU pipes: see zg_ex2_poly2; only the underflow side needs a clamp here
__device__ __forceinline__ zg_f2 zg_ex2_poly2_neg(zg_f2 x) {
    x.x = fmaxf(x.x, -126.f);
    x.y = fmaxf(x.y, -126.f);
    const zg_f2 r = zg_add2(x, zg_splat2(12582912.f));
    const zg_f2 xi = zg_add2(r, zg_splat2(-12582912.f));
    const zg_f2 f = zg_add2(x, zg_mul2(xi, zg_splat2(-1.f)));
    zg_f2 p = zg_splat2(0.001327647129073739f);
    p = zg_fma2(p, f, zg_splat2(0.009675540961325169f));
    p = zg_fma2(p, f, zg_splat2(0.05550713092088699f));
    p = zg_fma2(p, f, zg_splat2(0.24022120237350464f));
    p = zg_fma2(p, f, zg_splat2(0.6931469440460205f));
    p = zg_fma2(p, f, zg_splat2(1.0000001192092896f));
    p.x = __int_as_float(__float_as_int(p.x) + (__float_as_int(r.x) << 23));
    p.y = __int_as_float(__float_as_int(p.y) + (__float_as_int(r.y) << 23));
    return p;
}

template <typename T> __device__ __forceinline__ float2 pt_unpack2(uint32_t v);
template <> __device__ __forceinline__ float2 pt_unpack2<__nv_bfloat16>(uint32_t v) {
    return make_float2(__uint_as_float(v << 16), __uint_as_float(v & 0xffff0000u));
}
template <> __device__ __forceinline__ float2 pt_unpack2<__half>(uint32_t v) {
    return __half22float2(*reinterpret_cast<const __half2 *>(&v));
}
template <typename T> __device__ __forceinline__ uint32_t pt_pack2(float a, float b);
template <> __device__ __forceinline__ uint32_t pt_pack2<__nv_bfloat16>(float a, float b) {
    const __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t *>(&v);
}
template <> __device__ __forceinline__ uint32_t pt_pack2<__half>(float a, float b) {
    const __half2 v = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t *>(&v);
}

// softplus of a channel pair (reference threshold 20, selective_scan_fwd_kernel.cuh:153-156); numerics of zg_softplus20
__device__ __forceinline__ float2 pt_softplus20_2(float2 x) {
    float2 xm = make_float2(fminf(x.x, 20.f), fminf(x.y, 20.f));
    xm = zg_mul2(xm, zg_splat2(ZG_LOG2E));
    const float2 e = make_float2(zg_ex2(xm.x), zg_ex2(xm.y));
    float2 s = zg_fma2(e, zg_splat2(0.2f), zg_splat2(-0.25f));
    s = zg_fma2(e, s, zg_splat2(0.33333334f));
    s = zg_fma2(e, s, zg_splat2(-0.5f));
    s = zg_fma2(e, s, zg_splat2(1.f));
    s = zg_mul2(e, s);
    const float2 w = zg_add2(e, zg_splat2(1.f));
    const float2 lg = zg_mul2(make_float2(zg_lg2(w.x), zg_lg2(w.y)), zg_splat2(ZG_LN2));
    float2 r;
    r.x = (e.x < 0.03125f) ? s.x : lg.x;
    r.y = (e.y < 0.03125f) ? s.y : lg.y;
    r.x = (x.x > 20.f) ? x.x : r.x;
    r.y = (x.y > 20.f) ? x.y : r.y;
    return r;
}
// 1 / d for d in [1, 2^126] on the FMA pipe: integer-subtraction seed (relative error < 12.5 %) and three Newton steps in the
// residual form r += r (1 - d r); maximum relative error 6.8e-8 over the range (MUFU.RCP: 1.2e-7).
__device__ __forceinline__ float2 pt_rcp2_fma(float2 d) {
    float2 r = make_float2(__int_as_float(0x7EF311C7 - __float_as_int(d.x)), __int_as_float(0x7EF311C7 - __float_as_int(d.y)));
    const float2 nd = make_float2(-d.x, -d.y), one = zg_splat2(1.f);
#pragma unroll
    for (int i = 0; i < 3; ++i) r = zg_fma2(r, zg_fma2(nd, r, one), r);
    return r;
}
// SiLU of a channel pair.  ZG_SCAN_RCP_FMA: the reciprocal of the sigmoid on the FMA pipe instead of MUFU.RCP -- the scan kernels
// are bound by the MUFU pipe (20 per (b, e, l), one of them this reciprocal) and have issue slots to spare.  The exponent is
// clamped so that 1 + 2^t stays finite (z < -87: silu(z) ~ -1e-36 instead of -0).
#ifndef ZG_SCAN_RCP_FMA
#define ZG_SCAN_RCP_FMA 0
#endif
__device__ __forceinline__ float2 pt_silu2(float2 z) {
    float2 t = zg_mul2(z, zg_splat2(-ZG_LOG2E));
#if ZG_SCAN_RCP_FMA
    t.x = fminf(t.x, 126.f);
    t.y = fminf(t.y, 126.f);
    const float2 d = zg_add2(make_float2(zg_ex2(t.x), zg_ex2(t.y)), zg_splat2(1.f));
    return zg_mul2(z, pt_rcp2_fma(d));
#else
    const float2 d = zg_add2(make_float2(zg_ex2(t.x), zg_ex2(t.y)), zg_splat2(1.f));
    return zg_mul2(z, make_float2(zg_rcp(d.x), zg_rcp(d.y)));
#endif
}

__device__ __forceinline__ void pt_ldmatrix_x4(uint32_t &r0, uint32_t &r1, uint32_t &r2, uint32_t &r3, uint32_t saddr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(saddr));
}
__device__ __forceinline__ void pt_ldmatrix_x2(uint32_t &r0, uint32_t &r1, uint32_t saddr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0, %1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(saddr));
}
__device__ __forceinline__ void pt_ldmatrix_x1(uint32_t &r0, uint32_t saddr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x1.shared.b16 {%0}, [%1];" : "=r"(r0) : "r"(saddr));
}
// D(16x8, fp32) += A(16x16) B(16x8); rows 8..15 of A are zero here (a stage has 8 steps), so only d0, d1 carry data
template <typename T> __device__ __forceinline__ void pt_mma_k16(float &d0, float &d1, uint32_t a_lo, uint32_t a_hi, uint32_t b_lo, uint32_t b_hi) {
    float d2 = 0.f, d3 = 0.f;
    const uint32_t zero = 0u;
    if constexpr (sizeof(T) == 2 && std::is_same<T, __nv_bfloat16>::value) {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                     : "+f"(d0), "+f"(d1), "+f"(d2), "+f"(d3) : "r"(a_lo), "r"(zero), "r"(a_hi), "r"(zero), "r"(b_lo), "r"(b_hi));
    } else {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                     : "+f"(d0), "+f"(d1), "+f"(d2), "+f"(d3) : "r"(a_lo), "r"(zero), "r"(a_hi), "r"(zero), "r"(b_lo), "r"(b_hi));
    }
}
template <typename T> __device__ __forceinline__ void pt_mma_k8(float &d0, float &d1, uint32_t a, uint32_t b) {
    float d2 = 0.f, d3 = 0.f;
    const uint32_t zero = 0u;
    if constexpr (std::is_same<T, __nv_bfloat16>::value) {
        asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5}, {%6}, {%0, %1, %2, %3};"
                     : "+f"(d0), "+f"(d1), "+f"(d2), "+f"(d3) : "r"(a), "r"(zero), "r"(b));
    } else {
        asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5}, {%6}, {%0, %1, %2, %3};"
                     : "+f"(d0), "+f"(d1), "+f"(d2), "+f"(d3) : "r"(a), "r"(zero), "r"(b));
    }
}

// one stage (8 steps) of the recurrence for this thread's 16 / TPC states (NPAIR fp32x2 pairs); NP of the pairs use the FMA-pipe exp2.
// ddu_c: this channel's (delta', delta' u) pairs, one per step.  ypart: where this thread's partial y of step t goes (+ t * ypitch):
// with two threads per channel the two halves overwrite the pair they were computed from, else a separate tile.
// Software-pipelined by hand (ZG_SCAN_SWP, default on): ptxas emits the unrolled steps strictly one after the other
// (LDS -> multiplies -> 8 MUFU -> FMA chain -> STS, ~140 cycles of dependent latency per step and warp), so the decay factors
// exp2(delta' A) of step t + 1 -- which depend on nothing but (delta', A) -- are issued BEFORE the FMA part of step t.
template <int NP, int TPC, int PITCH = PT_F32ROW>
__device__ __forceinline__ void pt_main_stage(const unsigned char *__restrict__ ddu_c, const float *__restrict__ bcf_p, unsigned char *__restrict__ ypart, int ypitch,
                                              zg_f2 (&h2)[8 / TPC], const zg_f2 (&Al2p)[8 / TPC], bool store = true, int sync_step = -1, int bar_threads = 0) {
    constexpr int NPAIR = 8 / TPC, NQ = 4 / TPC;           // state pairs per thread; float4 loads of B (and of C) per step
    auto decay = [&](float dlx, zg_f2 (&a)[NPAIR]) {
        const zg_f2 dl = zg_splat2(dlx);
#pragma unroll
        for (int q = 0; q < NPAIR; ++q) {
            const zg_f2 x = zg_mul2(dl, Al2p[q]);
#if ZG_SCAN_EXP == 5
            a[q] = zg_add2(x, zg_splat2(1.f));              // experiment: everything but the exponentials
#else
            a[q] = (q < NP) ? zg_ex2_poly2_neg(x) : zg_ex2_mufu2(x);
#endif
        }
    };
#if ZG_SCAN_SWP
    zg_f2 a_cur[NPAIR];
    float2 dd = *reinterpret_cast<const float2 *>(ddu_c);
    decay(dd.x, a_cur);
#pragma unroll
    for (int t = 0; t < PT_TL; ++t) {
        const float4 *bc = reinterpret_cast<const float4 *>(bcf_p + t * 32);
        zg_f2 Bp[NPAIR], Cp[NPAIR];
#pragma unroll
        for (int k = 0; k < NQ; ++k) {
            const float4 Bk = bc[k], Ck = bc[4 + k];
            Bp[2 * k] = make_float2(Bk.x, Bk.y); Bp[2 * k + 1] = make_float2(Bk.z, Bk.w);
            Cp[2 * k] = make_float2(Ck.x, Ck.y); Cp[2 * k + 1] = make_float2(Ck.z, Ck.w);
        }
        const zg_f2 du = zg_splat2(dd.y);
        zg_f2 a_nxt[NPAIR];
        if (t + 1 < PT_TL) {                               // next step's pair and decays: in flight during this step's FMAs
            dd = *reinterpret_cast<const float2 *>(ddu_c + (t + 1) * PITCH);
            decay(dd.x, a_nxt);
        }
        zg_f2 y2 = zg_splat2(0.f);
#pragma unroll
        for (int q = 0; q < NPAIR; ++q) {
            h2[q] = zg_fma2(a_cur[q], h2[q], zg_mul2(du, Bp[q]));
            y2 = zg_fma2(Cp[q], h2[q], y2);
        }
        *reinterpret_cast<float *>(ypart + t * ypitch) = y2.x + y2.y;
        // staggered fairness barrier of the warp-private kernels (scan_fwd_wp.cuh): warp w of a CTA arrives after step w % 8
        if (t == sync_step) asm volatile("bar.sync 1, %0;" ::"r"(bar_threads) : "memory");
        if (t + 1 < PT_TL) {
#pragma unroll
            for (int q = 0; q < NPAIR; ++q) a_cur[q] = a_nxt[q];
        }
    }
#else
#pragma unroll
    for (int t = 0; t < PT_TL; ++t) {
        const float2 dd = *reinterpret_cast<const float2 *>(ddu_c + t * PITCH);      // (delta', delta' * u)
        const float4 *bc = reinterpret_cast<const float4 *>(bcf_p + t * 32);
        zg_f2 Bp[NPAIR], Cp[NPAIR];
#pragma unroll
        for (int k = 0; k < NQ; ++k) {
            const float4 Bk = bc[k], Ck = bc[4 + k];
            Bp[2 * k] = make_float2(Bk.x, Bk.y); Bp[2 * k + 1] = make_float2(Bk.z, Bk.w);
            Cp[2 * k] = make_float2(Ck.x, Ck.y); Cp[2 * k + 1] = make_float2(Ck.z, Ck.w);
        }
        const zg_f2 du = zg_splat2(dd.y);
        zg_f2 a[NPAIR];
        decay(dd.x, a);
        zg_f2 y2 = zg_splat2(0.f);
#pragma unroll
        for (int q = 0; q < NPAIR; ++q) {
            h2[q] = zg_fma2(a[q], h2[q], zg_mul2(du, Bp[q]));
            y2 = zg_fma2(Cp[q], h2[q], y2);
        }
        // (TPC == 2: both threads of the channel have read the pair -- one converged LDS -- before either overwrites its half)
#if ZG_SCAN_EXP == 3
        if (store) *reinterpret_cast<float *>(ypart + t * ypitch) = y2.x + y2.y;
#else
        *reinterpret_cast<float *>(ypart + t * ypitch) = y2.x + y2.y;
#endif
    }
#endif
}

struct PtMaps { CUtensorMap u, d, z; };    // (channels | x_dbl columns, seqlen, batch) tensor tiles of u, delta | x_dbl, z

__device__ __forceinline__ void pt_tma_load_3d(void *dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(zg_smem_u32(dst)),
                 "l"(map), "r"(zg_smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
// the thread's earlier cp.async copies arrive on `bar` when they land (the barrier's expected count includes this arrival)
__device__ __forceinline__ void pt_cp_async_arrive(uint64_t *bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(zg_smem_u32(bar)) : "memory");
}

// TPC threads per channel: 2 (16 / 2 = 8 states per thread, 128-thread CTAs, 9 CTAs / SM) is the product mapping; 4 (4 states per
// thread, 256-thread CTAs: twice the warps for the same instructions per (b, e, l)) is an experiment for under-occupied shapes
// (ZG_SCAN_TPC=4) that measured slower, see pt_launch_variant.
// PLAIN: the sampling / training call as the model makes it -- z gate present, softplus on, output in place and in order
// (no OUT_REVERSE / OUT_ACCUMULATE) -- with those choices compiled in: no uniform branches and no predicated-off accumulate code
// in the stage loop (post + pre 187 instead of ~250 SASS instructions; 0.502 vs 0.518 ms at config 2, same box, ZG_SCAN_PLAIN=0).
template <typename T, int R, int NPOLY, bool CKPT, int TPC = 2, bool PLAIN = false>
__global__ void __launch_bounds__(64 * TPC, TPC == 2 ? 9 : 6) scan_fwd_tma_kernel(const zg_scan_params p, const __grid_constant__ PtMaps maps) {
    static_assert(sizeof(T) == 2, "16-bit I/O only");
    static_assert(TPC == 2 || (TPC == 4 && R == 0 && NPOLY == 0), "four threads per channel: unfused, MUFU-only instantiation");
    using LY = PtLayout<R, TPC>;
    constexpr int PT_THREADS = 64 * TPC, NPAIR = 8 / TPC, NITEM = 4 / TPC;      // (step, channel pair) items per thread in pre / post
    constexpr bool FUSE = LY::FUSE;
    constexpr int NSTAGE = LY::NSTAGE, TL = PT_TL, CH = PT_CH, TILE = LY::TILE;
    extern __shared__ __align__(1024) unsigned char smem[];
    unsigned char *ddu = smem + LY::DDU_OFF;
    float *bcf = reinterpret_cast<float *>(smem + LY::BCF_OFF);
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + LY::BAR_OFF);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int part = tid % TPC;                                     // which 16 / TPC states of the channel
    const int E = p.dim, L = p.seqlen;
    const int per_group = E / p.ngroups;
    const int tiles_per_group = per_group / CH;
    const int tiles = tiles_per_group * p.ngroups;
    const int b = blockIdx.x / tiles;
    const int tile = blockIdx.x % tiles;
    const int g = tile / tiles_per_group;
    const int e0 = g * per_group + (tile % tiles_per_group) * CH;
    const int e = e0 + tid / TPC;                                   // main phase: this thread's channel
    const bool has_z = PLAIN ? true : (p.z != nullptr);
    const bool z_gather = has_z && p.z_rowmap != nullptr;           // z rows by cp.async through the table
    const bool softplus = PLAIN ? true : ((p.flags & ZG_SCAN_DELTA_SOFTPLUS) != 0);
    const int nstages = L / TL;

    // ---- per-thread constants -----------------------------------------------------------------------------------
    zg_f2 Al2p[NPAIR], h2[NPAIR];
    bool a_pos = false;
#pragma unroll
    for (int k = 0; k < NPAIR; ++k) {
        const float2 a = *reinterpret_cast<const float2 *>(p.A + (int64_t)e * 16 + 2 * NPAIR * part + 2 * k);
        Al2p[k] = zg_mul2(a, zg_splat2(ZG_LOG2E));
        a_pos = a_pos || a.x > 0.f || a.y > 0.f;
        h2[k] = zg_splat2(0.f);
    }
    // The two (step, channel pair) items a thread owns in the pre and post phases (same items in both: the post phase reads
    // the partial y from the 16 bytes its own pre phase filled, so a thread may run pre(s + 1) right after post(s)):
    //   unfused: lane = channel pair, steps warp and warp + 4  (128-byte coalesced output rows)
    //   fused:   step lane / 4, channel pairs 16 warp + 8 k + 2 (lane % 4) -- the m16n8 accumulator layout of the delta tile
    int it_swz[NITEM], it_ddu[NITEM];                      // byte offsets inside a swizzled 8 x 128 B tile / the fp32 pair tile
    float2 Dv[NITEM], biasv[NITEM];
#pragma unroll
    for (int k = 0; k < NITEM; ++k) {
        const int row = FUSE ? (lane >> 2) : warp + 2 * TPC * k;          // (2 TPC warps: rows warp, warp + 4 | row warp)
        const int pair = FUSE ? 8 * warp + 4 * k + (lane & 3) : lane;                  // channel pair 0..31 of the tile
        it_swz[k] = row * 128 + (((pair >> 2) ^ row) << 4) + (pair & 3) * 4;
        it_ddu[k] = row * PT_F32ROW + pair * 16;
        Dv[k] = p.D ? *reinterpret_cast<const float2 *>(p.D + e0 + 2 * pair) : make_float2(0.f, 0.f);
        biasv[k] = p.delta_bias ? *reinterpret_cast<const float2 *>(p.delta_bias + e0 + 2 * pair) : make_float2(0.f, 0.f);
    }

    // full[s]: one cp.async arrival per thread and stage (its gathered chunk, possibly none) + the TMA issuer's expect_tx
    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < NSTAGE; ++s) zg_mbar_init(&full[s], PT_THREADS + 1);
        zg_mbar_fence_init();
    }
    if constexpr (FUSE) {   // this CTA's 64 dt_proj rows -> shared memory (pitch WROW: conflict-free ldmatrix)
        constexpr int CPR = 2 * R / 16;   // 16-byte chunks per row
        const T *gw = reinterpret_cast<const T *>(p.dt_w) + (int64_t)e0 * p.dt_w_ld;
        for (int i = tid; i < CH * CPR; i += PT_THREADS) {
            const int row = i / CPR, ch = i % CPR;
            *reinterpret_cast<uint4 *>(smem + LY::W_OFF + row * LY::WROW + ch * 16) =
                *reinterpret_cast<const uint4 *>(gw + (int64_t)row * p.dt_w_ld + ch * 8);
        }
    }
    // NPOLY > 0 needs delta' A <= 0 (softplus'ed delta, non-positive A) for the one-sided clamp of the polynomial
    const bool use_poly = NPOLY > 0 && softplus && !__syncthreads_or(a_pos);
    __syncthreads();

    // ---- producer: thread 0 issues the tensor tiles; threads 64..127 gather one z chunk each, 64..95 a B|C chunk ----
    const uint32_t tx_bytes = TILE + (FUSE ? TL * LY::XBYTES : TILE) + ((has_z && !z_gather) ? TILE : 0);
    const int zr = (tid >> 3) & 7, zj = tid & 7;          // threads 64..127: z row / 16-byte column of the stage
    // batch element b of z: plain batch stride, or two-level (b / K, b % K) for the temporal video scan (zg_scan_params.z_batch_inner)
    const int64_t z_boff = p.z_batch_inner > 0 ? (int64_t)(b / p.z_batch_inner) * p.z_sb + (int64_t)(b % p.z_batch_inner) * p.z_sbi : (int64_t)b * p.z_sb;
    const unsigned char *zsrc = (z_gather && tid >= 64) ? reinterpret_cast<const unsigned char *>(reinterpret_cast<const T *>(p.z) + z_boff + e0 + zj * 8) : nullptr;
    const uint32_t z_sl2 = (uint32_t)p.z_sl * 2u;            // byte offsets inside a batch element fit 32 bits (host check)
    int zrow_next = (zsrc != nullptr) ? p.z_rowmap[zr] : 0;   // (permuted) source row of the NEXT stage to issue
    auto issue_stage = [&](int s, int slot) {             // all threads
        if (s >= nstages) return;
        unsigned char *sw = smem + LY::SWZ_OFF + slot * LY::NSWZ * TILE;
        unsigned char *xt = smem + LY::X_OFF + slot * LY::XSTAGE;
        uint64_t *bar = &full[slot];
        const int l0 = s * TL;
        if (tid == 0) {
            zg_mbar_expect_tx(bar, tx_bytes);
            pt_tma_load_3d(sw, &maps.u, bar, e0, l0, b);
            if (has_z && !z_gather) pt_tma_load_3d(sw + TILE, &maps.z, bar, e0, l0, b);
            if constexpr (FUSE) pt_tma_load_3d(xt, &maps.d, bar, 0, l0, b);
            else pt_tma_load_3d(sw + 2 * TILE, &maps.d, bar, e0, l0, b);
        }
        if (tid >= 64) {
            if (zsrc != nullptr) {                        // chunk (row zr, column zj) lands swizzled like the TMA tiles
                zg_cp_async16(sw + TILE + zr * 128 + ((zj ^ zr) << 4), zsrc + (uint32_t)zrow_next * z_sl2);
                const int ln = l0 + TL + zr;
                zrow_next = (ln < L) ? p.z_rowmap[ln] : 0;
            }
            if (!FUSE && tid < 96) {                      // raw B | C rows: 8 steps x (2 + 2) chunks
                const int r = (tid >> 2) & 7, w = (tid >> 1) & 1, j = tid & 1;
                const T *src = w ? reinterpret_cast<const T *>(p.C) + (int64_t)b * p.C_sb + (int64_t)g * p.C_sg + (int64_t)(l0 + r) * p.C_sl
                                 : reinterpret_cast<const T *>(p.B) + (int64_t)b * p.B_sb + (int64_t)g * p.B_sg + (int64_t)(l0 + r) * p.B_sl;
                zg_cp_async16(xt + r * 64 + w * 32 + j * 16, src + j * 8);
            }
        }
        pt_cp_async_arrive(bar);
    };
#pragma unroll
    for (int s = 0; s < NSTAGE; ++s) issue_stage(s, s);

    // ---- pre / post work of a thread's two items.  post(s) and pre(s + 1) run in the same barrier interval and touch the same
    // 16 bytes of the pair tile (y read, then (delta', delta' u) written), so they are interleaved item by item: four
    // independent MUFU chains (SiLU of two items, softplus of two items) per thread instead of two after two.
    auto bc_convert = [&](const unsigned char *xt) {      // B | C rows -> fp32 [step][B0..15 C0..15]: one 16-bit pair per thread
        if (TPC > 2 && tid >= 128) return;
        const int t = tid >> 4, j = tid & 15;
        const uint32_t raw = FUSE ? *reinterpret_cast<const uint32_t *>(xt + t * LY::XBYTES + 2 * R + j * 4)
                                  : *reinterpret_cast<const uint32_t *>(xt + t * 64 + j * 4);
        *reinterpret_cast<float2 *>(bcf + t * 32 + 2 * j) = pt_unpack2<T>(raw);
    };
    // raw (rounded) delta of the thread's two items: from the delta tile, or (fused) from the tensor-core product
    //     x_dbl[8 steps, 0:R] . W[64 ch, 0:R]^T      (this warp: channels 16 warp .. +15; rows 8..15 of the m16 tile are zero)
    auto delta_items = [&](const unsigned char *sw, const unsigned char *xt, float2 (&dlt)[NITEM]) {
        if constexpr (FUSE) {
            const uint32_t xs = zg_smem_u32(xt), ws = zg_smem_u32(smem + LY::W_OFF);
            float d[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
            const uint32_t a_addr = xs + (lane & 7) * LY::XBYTES + (lane >> 3) * 16;
            const uint32_t b_addr = ws + (16 * warp + (lane & 7) + 8 * (lane >> 4)) * LY::WROW + ((lane >> 3) & 1) * 16;
#pragma unroll
            for (int k2 = 0; k2 < R / 32; ++k2) {           // two k16 steps per iteration
                uint32_t a0, a1, a2, a3, b0, b1, b2, b3;
                pt_ldmatrix_x4(a0, a1, a2, a3, a_addr + 64 * k2);
                pt_ldmatrix_x4(b0, b1, b2, b3, b_addr + 64 * k2);
                pt_mma_k16<T>(d[0][0], d[0][1], a0, a1, b0, b1);
                pt_mma_k16<T>(d[1][0], d[1][1], a0, a1, b2, b3);
                pt_ldmatrix_x4(b0, b1, b2, b3, b_addr + 64 * k2 + 32);
                pt_mma_k16<T>(d[0][0], d[0][1], a2, a3, b0, b1);
                pt_mma_k16<T>(d[1][0], d[1][1], a2, a3, b2, b3);
            }
            constexpr int KREM = R % 32;                    // 0, 8, 16 or 24 columns left
            constexpr int KB = (R / 32) * 64;               // their byte offset in a row
            if constexpr (KREM >= 16) {
                uint32_t a0, a1, b0, b1, b2, b3;
                pt_ldmatrix_x2(a0, a1, xs + (lane & 7) * LY::XBYTES + ((lane >> 3) & 1) * 16 + KB);
                pt_ldmatrix_x4(b0, b1, b2, b3, b_addr + KB);
                pt_mma_k16<T>(d[0][0], d[0][1], a0, a1, b0, b1);
                pt_mma_k16<T>(d[1][0], d[1][1], a0, a1, b2, b3);
            }
            if constexpr (KREM % 16 == 8) {
                constexpr int KB8 = KB + (KREM >= 16 ? 32 : 0);
                uint32_t a0, b0, b1;
                pt_ldmatrix_x1(a0, xs + (lane & 7) * LY::XBYTES + KB8);
                pt_ldmatrix_x2(b0, b1, ws + (16 * warp + (lane & 7) + 8 * ((lane >> 3) & 1)) * LY::WROW + KB8);
                pt_mma_k8<T>(d[0][0], d[0][1], a0, b0);
                pt_mma_k8<T>(d[1][0], d[1][1], a0, b1);
            }
            // round like the reference's GEMM output (selective_scan_interface.py:323 produces delta in the I/O dtype)
#pragma unroll
            for (int j = 0; j < 2; ++j) dlt[j] = pt_unpack2<T>(pt_pack2<T>(d[j][0], d[j][1]));
        } else {
#pragma unroll
            for (int k = 0; k < NITEM; ++k) dlt[k] = pt_unpack2<T>(*reinterpret_cast<const uint32_t *>(sw + 2 * TILE + it_swz[k]));
        }
    };
    auto pre_item = [&](int k, float2 dl, const unsigned char *sw) {     // bias, softplus, * u -> (delta', delta' u) pairs
        dl = zg_add2(dl, biasv[k]);
#if ZG_SCAN_EXP == 1
        if (softplus) dl = zg_mul2(dl, dl);
#else
        if (softplus) dl = pt_softplus20_2(dl);
#endif
        const float2 du = zg_mul2(dl, pt_unpack2<T>(*reinterpret_cast<const uint32_t *>(sw + it_swz[k])));
        float2 *dst = reinterpret_cast<float2 *>(ddu + it_ddu[k]);
        dst[0] = make_float2(dl.x, du.x);
        dst[1] = make_float2(dl.y, du.y);
    };
    // output rows: step l -> sequence position l, or seqlen - 1 - l (ZG_SCAN_OUT_REVERSE: the backward sweep of scan_type v2)
    const bool out_rev = PLAIN ? false : ((p.flags & ZG_SCAN_OUT_REVERSE) != 0), out_acc = PLAIN ? false : ((p.flags & ZG_SCAN_OUT_ACCUMULATE) != 0);
    const int64_t out_row = out_rev ? -p.out_sl : p.out_sl;
    const int r0 = FUSE ? (lane >> 2) : warp;               // the thread's first row of a stage
    const int64_t out_step = FUSE ? 8 : 4 * out_row;      // element distance between the thread's two output pairs (TPC == 2)
    T *gout = reinterpret_cast<T *>(p.out) + (int64_t)b * p.out_sb + (int64_t)(out_rev ? L - 1 - r0 : r0) * p.out_sl + e0 +
              (FUSE ? 16 * warp + 2 * (lane & 3) : 2 * lane);
    const int64_t out_stage = (int64_t)TL * out_row;
    auto post_item = [&](int k, const unsigned char *sw) {               // y = y_lo + y_hi + D u, SiLU(z) gate, store
        float2 ysum;
        if constexpr (TPC == 2) {
            const float4 yy = *reinterpret_cast<const float4 *>(ddu + it_ddu[k]);   // (lo, hi) halves of 2 channels
            ysum = zg_add2(make_float2(yy.x, yy.z), make_float2(yy.y, yy.w));
        } else {                                          // 4 partial sums per channel in the separate y tile
            const float4 *yp = reinterpret_cast<const float4 *>(smem + LY::Y_OFF + (it_ddu[k] / PT_F32ROW) * LY::YROW + ((it_ddu[k] % PT_F32ROW) / 16) * 32);
            const float4 a4 = yp[0], b4 = yp[1];
            ysum = make_float2((a4.x + a4.y) + (a4.z + a4.w), (b4.x + b4.y) + (b4.z + b4.w));
        }
        const float2 u2 = pt_unpack2<T>(*reinterpret_cast<const uint32_t *>(sw + it_swz[k]));
        float2 y = zg_fma2(Dv[k], u2, ysum);
#if ZG_SCAN_EXP == 1
        if (has_z) y = zg_mul2(y, pt_unpack2<T>(*reinterpret_cast<const uint32_t *>(sw + TILE + it_swz[k])));
#else
        if (has_z) y = zg_mul2(y, pt_silu2(pt_unpack2<T>(*reinterpret_cast<const uint32_t *>(sw + TILE + it_swz[k]))));
#endif
        uint32_t *dst = reinterpret_cast<uint32_t *>(gout + (k ? out_step : 0));
        if (out_acc) {      // out = round(out + round(y)): the eager sum of two I/O-dtype tensors (mamba_simple.py:337)
            const float2 prev = pt_unpack2<T>(*dst), yr = pt_unpack2<T>(pt_pack2<T>(y.x, y.y));
            y = zg_add2(prev, yr);
        }
        *dst = pt_pack2<T>(y.x, y.y);
    };

    // ---- the pipeline ------------------------------------------------------------------------------------------------
    const unsigned char *ddu_c = ddu + (tid / TPC) * 8;
    const float *bcf_p = bcf + 2 * NPAIR * part;
    unsigned char *ypart = TPC == 2 ? ddu + (tid / TPC) * 8 + part * 4 : smem + LY::Y_OFF + (tid / TPC) * 16 + part * 4;
    constexpr int ypitch = TPC == 2 ? PT_F32ROW : LY::YROW;
    {   // stage 0: pre only
        const unsigned char *sw = smem + LY::SWZ_OFF, *xt = smem + LY::X_OFF;
        zg_mbar_wait(&full[0], 0);
        float2 dlt[NITEM];
        delta_items(sw, xt, dlt);
#pragma unroll
        for (int k = 0; k < NITEM; ++k) pre_item(k, dlt[k], sw);
        bc_convert(xt);
    }
    __syncthreads();
    int slot = 0, nslot = 1;
    uint32_t npar = 0;                                       // phase parity of the next stage's slot
    for (int s = 0; s < nstages; ++s) {
        if (NPOLY > 0 && use_poly) pt_main_stage<NPOLY, TPC>(ddu_c, bcf_p, ypart, ypitch, h2, Al2p);
        else pt_main_stage<0, TPC>(ddu_c, bcf_p, ypart, ypitch, h2, Al2p, s == nstages - 1);
        if constexpr (CKPT) {       // recompute seeds of the backward: state after every 8 steps, (batch, n_ckpt, dim, dstate)
            float4 *dst = reinterpret_cast<float4 *>(p.ckpt + (((int64_t)b * (L >> 3) + s) * E + e) * 16 + 2 * NPAIR * part);
#pragma unroll
            for (int k = 0; k < NPAIR / 2; ++k) dst[k] = make_float4(h2[2 * k].x, h2[2 * k].y, h2[2 * k + 1].x, h2[2 * k + 1].y);
        }
        const unsigned char *sw = smem + LY::SWZ_OFF + slot * LY::NSWZ * TILE;
        const unsigned char *swn = smem + LY::SWZ_OFF + nslot * LY::NSWZ * TILE;
        const unsigned char *xtn = smem + LY::X_OFF + nslot * LY::XSTAGE;
#if ZG_SCAN_EXP == 2 || ZG_SCAN_EXP == 3
        if (s == nstages - 1) { for (int k = 0; k < NITEM; ++k) post_item(k, sw); }   // experiment: the recurrence alone
#else
        __syncthreads();            // y complete; B/C tile free
        if (s + 1 < nstages) {      // post(s) interleaved with pre(s + 1)
            zg_mbar_wait(&full[nslot], npar);
            float2 dlt[NITEM];
            delta_items(swn, xtn, dlt);
#pragma unroll
            for (int k = 0; k < NITEM; ++k) { post_item(k, sw); pre_item(k, dlt[k], swn); }
            bc_convert(xtn);
        } else {
#pragma unroll
            for (int k = 0; k < NITEM; ++k) post_item(k, sw);
        }
        gout += out_stage;
        __syncthreads();            // raw slot of stage s free; tiles of stage s + 1 complete
        issue_stage(s + NSTAGE, slot);
#endif
        slot = nslot;
        if (++nslot == NSTAGE) { nslot = 0; npar ^= 1; }
    }
    if (p.last_state) {
        float4 *dst = reinterpret_cast<float4 *>(p.last_state + ((int64_t)b * E + e) * 16 + 2 * NPAIR * part);
#pragma unroll
        for (int k = 0; k < NPAIR / 2; ++k) dst[k] = make_float4(h2[2 * k].x, h2[2 * k].y, h2[2 * k + 1].x, h2[2 * k + 1].y);
    }
}

inline int pt_env_int(const char *name, int dflt) {
    const char *e = getenv(name);
    return e ? atoi(e) : dflt;
}

typedef CUresult (*PtEncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                    const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline PtEncodeTiledFn pt_get_encode() {
    static PtEncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PtEncodeTiledFn>(p);
    }
    return fn;
}
// (cols, seqlen, batch) view of a token-major 16-bit tensor -> tensor map with a (box_cols x 8 steps x 1) box, rows dense in smem
// (cols, seqlen, batch) view of a token-major 16-bit tensor -> tensor map with a (box_cols x 8 steps x 1) box.
// swizzle: the 64-channel tiles use the 128-byte swizzle (rows of exactly 128 B), the x_dbl rows land dense.
template <typename T>
inline int pt_make_map(CUtensorMap *m, const void *base, int64_t cols, int64_t seqlen, int64_t batch, int64_t sl, int64_t sb, int box_cols, bool swizzle) {
    PtEncodeTiledFn enc = pt_get_encode();
    if (!enc) return zg_set_error("scan_fwd(tma): cuTensorMapEncodeTiled not available from the driver");
    cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)seqlen, (cuuint64_t)batch};
    cuuint64_t strides[2] = {(cuuint64_t)sl * 2, (cuuint64_t)(batch > 1 ? sb : sl * seqlen) * 2};
    cuuint32_t box[3] = {(cuuint32_t)box_cols, (cuuint32_t)PT_TL, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    const CUtensorMapDataType dt = std::is_same<T, __nv_bfloat16>::value ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    CUresult r = enc(m, dt, 3, const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     swizzle ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return -1;        // not expressible as a tensor map (stride limits): the caller falls back to the round-1 kernel
    return 0;
}

template <typename T, int R, int NPOLY, bool CKPT, int TPC = 2, bool PLAIN = false> int pt_launch(const zg_scan_params &p, cudaStream_t stream) {
    if constexpr (!PLAIN && R == 0 && TPC == 2) {     // the model's own call: the specialised instantiation (ZG_SCAN_PLAIN=0: A/B timing)
        static const bool plain_ok = [] { const char *e = getenv("ZG_SCAN_PLAIN"); return !(e && e[0] == '0'); }();
        if (plain_ok && p.z && (p.flags & ZG_SCAN_DELTA_SOFTPLUS) && !(p.flags & (ZG_SCAN_OUT_REVERSE | ZG_SCAN_OUT_ACCUMULATE)))
            return pt_launch<T, R, NPOLY, CKPT, TPC, true>(p, stream);
    }
    using LY = PtLayout<R, TPC>;
    PtMaps maps;
    memset(&maps, 0, sizeof(maps));
    int rc = pt_make_map<T>(&maps.u, p.u, p.dim, p.seqlen, p.batch, p.u_sl, p.u_sb, PT_CH, true);
    if (!rc) rc = R > 0 ? pt_make_map<T>(&maps.d, p.dt_x, R + 32, p.seqlen, p.batch, p.dt_x_sl, p.dt_x_sb, R + 32, false)
                        : pt_make_map<T>(&maps.d, p.delta, p.dim, p.seqlen, p.batch, p.delta_sl, p.delta_sb, PT_CH, true);
    if (!rc && p.z && !p.z_rowmap) rc = pt_make_map<T>(&maps.z, p.z, p.dim, p.seqlen, p.batch, p.z_sl, p.z_sb, PT_CH, true);
    if (rc) return rc;
    auto kern = scan_fwd_tma_kernel<T, R, NPOLY, CKPT, TPC, PLAIN>;
    static bool attr_dev[64] = {};      // per instantiation and device
    int dev = 0;
    cudaGetDevice(&dev);
    if (!attr_dev[dev & 63]) {
        cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, LY::TOTAL);
        if (err != cudaSuccess) return zg_set_error("scan_fwd(tma): cudaFuncSetAttribute(%d B smem): %s", LY::TOTAL, cudaGetErrorString(err));
        cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        attr_dev[dev & 63] = true;
    }
    const long long nblk = (long long)(p.dim / PT_CH) * p.batch;
    kern<<<(unsigned)nblk, 64 * TPC, LY::TOTAL, stream>>>(p, maps);
    zg_count_launch();
    zg_note_scan_kernel(R > 0 ? "zg::scan_fwd_tma_kernel (CTA-wide phases, TMA tensor tiles, fused dt_proj prologue)" : "zg::scan_fwd_tma_kernel (CTA-wide phases, TMA tensor tiles)");
    return zg_check_launch("scan_fwd(tma)");
}

template <typename T, int R> int pt_launch_variant(const zg_scan_params &p, cudaStream_t stream) {
    static int npoly = -1;
    if (npoly < 0) { npoly = pt_env_int("ZG_SCAN_TMA_NPOLY", ZG_SCAN_TMA_NPOLY_DEFAULT); if (npoly < 0 || npoly > 2) npoly = 0; }
    if constexpr (R == 0) {
        // ZG_SCAN_TPC=4: four threads per channel (twice the warps for the same work).  Opt-in only: measured SLOWER than two at
        // every under-occupied shape it was meant for (bs 32, L 4096, E 1536: 1.72 vs 1.46 ms; bs 16, L 1024, E 1280: 0.249 vs
        // 0.224 ms) -- eight warps per barrier cost more than the extra warps hide -- and a batch-size dependent choice would
        // make results depend on the batch split (the partial sums of y associate differently).
        static int tpc_env = -1;
        if (tpc_env < 0) tpc_env = pt_env_int("ZG_SCAN_TPC", 2);
        if (tpc_env == 4) return p.ckpt ? pt_launch<T, 0, 0, true, 4>(p, stream) : pt_launch<T, 0, 0, false, 4>(p, stream);
    }
    if (p.ckpt) return pt_launch<T, R, 0, true>(p, stream);        // training forward (writes the recompute seeds)
    if (npoly == 1) return pt_launch<T, R, 1, false>(p, stream);
    if (npoly == 2) return pt_launch<T, R, 2, false>(p, stream);
    return pt_launch<T, R, 0, false>(p, stream);
}

// warp-private pipeline (scan_fwd_wp.cuh), compiled in its own translation units
int scan_fwd_wp_bf16(const zg_scan_params &p, cudaStream_t stream, int mode);
int scan_fwd_wp_f16(const zg_scan_params &p, cudaStream_t stream, int mode);
int scan_fwd_wp2_bf16(const zg_scan_params &p, cudaStream_t stream, int mode);     // two channels per lane (scan_fwd_wp2.cuh)
int scan_fwd_wp2_f16(const zg_scan_params &p, cudaStream_t stream, int mode);
int scan_fwd_wph_bf16(const zg_scan_params &p, cudaStream_t stream, int nd, int ns);   // mixed 32- / 16-channel warps (scan_fwd_wph.cuh)
int scan_fwd_wph_f16(const zg_scan_params &p, cudaStream_t stream, int nd, int ns);
template <typename T> inline int wp_dispatch(const zg_scan_params &p, cudaStream_t stream, int mode, int nd = 0, int ns = 0) {
    if constexpr (std::is_same<T, __nv_bfloat16>::value)
        return mode == 5 ? scan_fwd_wph_bf16(p, stream, nd, ns) : mode >= 3 ? scan_fwd_wp2_bf16(p, stream, mode) : scan_fwd_wp_bf16(p, stream, mode);
    else
        return mode == 5 ? scan_fwd_wph_f16(p, stream, nd, ns) : mode >= 3 ? scan_fwd_wp2_f16(p, stream, mode) : scan_fwd_wp_f16(p, stream, mode);
}

// Which hot-path kernel runs a call (ZG_SCAN_WP unset).  All of them compute the same bits; what differs is how the work
// quantises over the 4 x SMs sub-partitions and how busy each keeps its MUFU pipe (thresholds carried over from a 148-SM GPU, expressed per SM; not re-tuned on H100):
// the 32-channel warps of scan_fwd_wp2 reach 85 % of the pipe against 76-79 % for 16-channel warps, but their unit of work is twice
// as large.  In 16-channel units, with U of them and S SMs, the fullest sub-partition carries
//     CTA-wide kernel (4 warps, one per sub-partition)      ceil(ceil(U / 4) / S)
//     32-channel warps                                      2 ceil(ceil(ceil(U / 2) / S) / 4)
//     mixed CTAs, two per SM, nd wide + ns narrow warps     nd / 4 * 2 + ns / 2   per CTA pair: (2 nd + ns) / 2
// Several waves: 32-channel warps (finished CTAs are replaced, the quantisation does not matter; measured - 5 %).  One wave: the
// 32-channel warps when they quantise no worse than the CTA-wide kernel (FacesHQ-1024 layer shape: 6 = 6, measured - 7 %), else
// mixed CTAs when those do (config 2: U = 5120 -> 18 units per CTA = 8 + 2 warps, 9 = 9, measured - 8 %), else the CTA-wide kernel
// (batch 16: 3 against 4).  The training forward (checkpoints) keeps the CTA-wide kernel.
inline ScanChoice scan_auto_choice(const zg_scan_params &p) {
    static int sms_dev[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (!sms_dev[dev & 63]) cudaDeviceGetAttribute(&sms_dev[dev & 63], cudaDevAttrMultiProcessorCount, dev);
    return scan_choice_for((long long)(p.dim / 16) * p.batch, sms_dev[dev & 63] > 0 ? sms_dev[dev & 63] : 132, p.ckpt != nullptr);
}

// host-side eligibility test + launch; returns -1 when the call does not fit the specialisation (never for a fused request:
// that one is an error, reported through zg_set_error with a positive return code)
template <typename T> int try_launch_scan_fwd_tma(const zg_scan_params &p, cudaStream_t stream) {
    const bool fuse = p.dt_w != nullptr;
    auto decline = [&](const char *why) -> int {
        if (fuse) return zg_set_error("selective_scan_fwd: fused dt_proj prologue not applicable: %s", why);
        return -1;
    };
    static int enabled = -1;
    if (enabled < 0) enabled = pt_env_int("ZG_SCAN_TMA", 1);
    if (!enabled && !fuse) return -1;
    if (sizeof(T) != 2) return decline("needs 16-bit I/O");
    const bool varBC = (p.flags & ZG_SCAN_VARIABLE_B) && (p.flags & ZG_SCAN_VARIABLE_C);
    if (!varBC || p.dstate != 16) return decline("needs input-dependent B and C with dstate 16");
    if (p.seqlen % PT_TL != 0 || p.seqlen == 0) return decline("seqlen must be a multiple of 8");
    if (p.ckpt && p.ckpt_every != 8) return decline("checkpoints every 8 steps only");
    if ((p.dim / p.ngroups) % PT_CH != 0) return decline("dim / groups must be a multiple of 64");
    if (!(p.u_sd == 1 && p.out_sd == 1 && (!p.z || p.z_sd == 1) && p.B_sn == 1 && p.C_sn == 1) || (!fuse && p.delta_sd != 1))
        return decline("needs the dim-contiguous (token-major) layout");
    uintptr_t al = reinterpret_cast<uintptr_t>(p.u) | reinterpret_cast<uintptr_t>(p.z) | reinterpret_cast<uintptr_t>(p.B) |
                   reinterpret_cast<uintptr_t>(p.C) | reinterpret_cast<uintptr_t>(p.ckpt) | reinterpret_cast<uintptr_t>(p.last_state);
    int64_t so = p.u_sb | (p.z ? (p.z_sb | p.z_sl) : 0) | p.B_sb | p.B_sg | p.C_sb | p.C_sg | p.u_sl | p.B_sl | p.C_sl;
    if (!fuse) { al |= reinterpret_cast<uintptr_t>(p.delta); so |= p.delta_sb | p.delta_sl; }
    else { al |= reinterpret_cast<uintptr_t>(p.dt_w) | reinterpret_cast<uintptr_t>(p.dt_x); so |= p.dt_w_ld | p.dt_x_sb | p.dt_x_sl; }
    if (al % 16 != 0 || so % 8 != 0) return decline("rows must be 16-byte aligned");
    if (reinterpret_cast<uintptr_t>(p.out) % 4 != 0 || (p.out_sb | p.out_sl) % 2 != 0) return decline("output rows must be 4-byte aligned");
    if ((reinterpret_cast<uintptr_t>(p.A) | reinterpret_cast<uintptr_t>(p.D) | reinterpret_cast<uintptr_t>(p.delta_bias)) % 8 != 0) return decline("A / D / delta_bias must be 8-byte aligned");
    const int64_t lim = 0x7fffffffLL;   // byte offsets inside one batch element fit 32 bits
    if ((int64_t)p.seqlen * p.u_sl * 2 > lim || (!fuse && (int64_t)p.seqlen * p.delta_sl * 2 > lim) || (p.z && (int64_t)p.seqlen * p.z_sl * 2 > lim))
        return decline("batch element too large for 32-bit offsets");
    if ((long long)(p.dim / PT_CH) * p.batch > 0x7fffffffLL) return decline("grid too large");
    if (p.z_batch_inner > 0 && (!p.z || !p.z_rowmap || p.z_sbi % 8 != 0)) return decline("z_batch_inner needs z with a z_rowmap and 16-byte aligned rows");
    if (!fuse) {
        // ZG_SCAN_WP: the warp-private pipelines: 1 / 2 = scan_fwd_wp.cuh (one channel per lane; cp.async staging / TMA tiles for
        // u and delta), 3 / 4 = scan_fwd_wp2.cuh (two channels per lane; cp.async / TMA), 5 = scan_fwd_wph.cuh (mixed warps), 0 = this file's kernel
        // (read at every call, unlike the other switches: the tests compare the kernels bit for bit inside one process)
        const int wp_mode = pt_env_int("ZG_SCAN_WP", ZG_SCAN_WP_DEFAULT);
        if (wp_mode >= 1 && wp_mode <= 5) return wp_dispatch<T>(p, stream, wp_mode);
        if (wp_mode < 0) {
            const ScanChoice c = scan_auto_choice(p);
            if (c.mode) return wp_dispatch<T>(p, stream, c.mode, c.nd, c.ns);
        }
        return pt_launch_variant<T, 0>(p, stream);
    }
    // fused prologue: B and C must be the tail of the dt_x rows (the x_dbl rows of x_proj)
    const T *x = reinterpret_cast<const T *>(p.dt_x);
    if (p.ngroups != 1 || reinterpret_cast<const T *>(p.B) != x + p.dt_rank || reinterpret_cast<const T *>(p.C) != x + p.dt_rank + 16 ||
        p.B_sb != p.dt_x_sb || p.C_sb != p.dt_x_sb || p.B_sl != p.dt_x_sl || p.C_sl != p.dt_x_sl)
        return decline("B and C must be columns dt_rank .. dt_rank + 31 of the dt_x rows (one group)");
    if ((int64_t)p.seqlen * p.dt_x_sl * 2 > lim) return decline("batch element too large for 32-bit offsets");
    switch (p.dt_rank) {
        case 40: return pt_launch_variant<T, 40>(p, stream);
        case 48: return pt_launch_variant<T, 48>(p, stream);
        default: return decline("dt_rank must be 40 or 48 in this build (embed_dim 640 / 768)");
    }
}

}  // namespace zg
