// Depthwise causal conv1d (+bias, +SiLU) forward / backward for sm_90a.
//
// Replaces causal_conv1d_fwd_kernel / causal_conv1d_channellast_fwd_kernel and their backward
// (dis_causal_conv1d/csrc/causal_conv1d_fwd.cu:39-158,193-330, causal_conv1d_bwd.cu:46-505).
// HBM-bound elementwise work: one 16-byte vector per thread per step, fully coalesced, fp32 math.
//   dim-contiguous ("channel last", token major): a thread owns VEC adjacent channels and slides
//     down LCH consecutive tokens with the W-1 previous inputs in registers; optional x_rowmap
//     gathers the input ROWS through the zigzag permutation (whole 2E*2-byte rows are contiguous,
//     so the gather is free: it only changes which row address is loaded).
//   seq-contiguous ("channel first", reference layout): a thread owns VEC consecutive positions of
//     one (batch, channel) row and reads the preceding vector for the halo.
#include "zg_common.cuh"
#include <stdlib.h>
#include <type_traits>

namespace zg {

constexpr int CONV_LCH = 32;   // tokens per thread, dim-contiguous kernels
constexpr int CONV_RB = 8;     // rows fetched per batch of independent loads

template <typename T, int VEC> struct VecT;  // VEC elements of T
template <typename T> struct VecT<T, 1> { T e[1]; };
template <> struct alignas(16) VecT<float, 4> { float e[4]; };
template <> struct alignas(16) VecT<__half, 8> { __half e[8]; };
template <> struct alignas(16) VecT<__nv_bfloat16, 8> { __nv_bfloat16 e[8]; };
template <> struct alignas(4) VecT<__half, 2> { __half e[2]; };
template <> struct alignas(4) VecT<__nv_bfloat16, 2> { __nv_bfloat16 e[2]; };
template <> struct alignas(8) VecT<float, 2> { float e[2]; };
template <> struct alignas(8) VecT<__half, 4> { __half e[4]; };
template <> struct alignas(8) VecT<__nv_bfloat16, 4> { __nv_bfloat16 e[4]; };

template <typename T, int VEC>
__device__ __forceinline__ void load_vec(float (&dst)[VEC], const T *src) {
    VecT<T, VEC> v = *reinterpret_cast<const VecT<T, VEC> *>(src);
#pragma unroll
    for (int i = 0; i < VEC; ++i) dst[i] = zg_to_float<T>(v.e[i]);
}
template <typename T, int VEC>
__device__ __forceinline__ void store_vec(T *dst, const float (&src)[VEC]) {
    VecT<T, VEC> v;
#pragma unroll
    for (int i = 0; i < VEC; ++i) v.e[i] = zg_from_float<T>(src[i]);
    *reinterpret_cast<VecT<T, VEC> *>(dst) = v;
}

template <typename W> __device__ __forceinline__ float load_w(const void *p, int64_t i) {
    return zg_to_float<W>(reinterpret_cast<const W *>(p)[i]);
}
__device__ __forceinline__ float load_w_dt(const void *p, int64_t i, int wdtype) {
    if (wdtype == ZG_F32) return load_w<float>(p, i);
    if (wdtype == ZG_F16) return load_w<__half>(p, i);
    return load_w<__nv_bfloat16>(p, i);
}

// ------------------------------------------------------------------------------------------------
// forward, dim-contiguous
template <typename T, int VEC>
__global__ void __launch_bounds__(128, 5) conv_fwd_dimc_kernel(const zg_conv_params p) {
    const int E = p.dim, L = p.seqlen, W = p.width;
    const int nvec = (E + VEC - 1) / VEC;
    const int nchunk = (L + CONV_LCH - 1) / CONV_LCH;
    const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (int64_t)p.batch * nchunk * nvec) return;
    const int v = (int)(gid % nvec);
    const int ch = (int)((gid / nvec) % nchunk);
    const int b = (int)(gid / ((int64_t)nvec * nchunk));
    const int e0 = v * VEC;
    const int l0 = ch * CONV_LCH;
    const T *x = reinterpret_cast<const T *>(p.x) + (int64_t)b * p.x_sb + e0;
    T *out = reinterpret_cast<T *>(p.out) + (int64_t)b * p.out_sb + e0;

    float w[4][VEC], bias[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
        const bool ok = e0 + i < E;
        bias[i] = (p.bias && ok) ? load_w_dt(p.bias, e0 + i, p.wdtype) : 0.f;
#pragma unroll
        for (int k = 0; k < 4; ++k)   // w[k] multiplies x[l - k]  (weight index W-1-k)
            w[k][i] = (ok && k < W) ? load_w_dt(p.weight, (int64_t)(e0 + i) * W + (W - 1 - k), p.wdtype) : 0.f;
    }
    // rows are fetched in batches of CONV_RB: all CONV_RB 16-byte loads are issued before the first one is
    // consumed (memory-level parallelism; the kernel streams ~335 MB per call at BASELINE config 2)
    auto row_ptr = [&](int l) -> const T * {
        const int64_t row = p.x_rowmap ? p.x_rowmap[l] : l;
        return x + row * p.x_sl;
    };
    auto load_row = [&](int l, float (&dst)[VEC]) {
        if (l < 0 || l >= L) {
#pragma unroll
            for (int i = 0; i < VEC; ++i) dst[i] = 0.f;
            return;
        }
        load_vec<T, VEC>(dst, row_ptr(l));
    };
    float x1[VEC], x2[VEC], x3[VEC];   // x[l-1], x[l-2], x[l-3]
    load_row(l0 - 1, x1);
    load_row(l0 - 2, x2);
    load_row(l0 - 3, x3);
    const int lend = min(l0 + CONV_LCH, L);
    for (int lb = l0; lb < lend; lb += CONV_RB) {
        VecT<T, VEC> raw[CONV_RB];
#pragma unroll
        for (int j = 0; j < CONV_RB; ++j)
            if (lb + j < lend) raw[j] = *reinterpret_cast<const VecT<T, VEC> *>(row_ptr(lb + j));
#pragma unroll
        for (int j = 0; j < CONV_RB; ++j) {
            if (lb + j < lend) {
                float o[VEC];
#pragma unroll
                for (int i = 0; i < VEC; ++i) {
                    const float x0 = zg_to_float<T>(raw[j].e[i]);
                    float acc = bias[i];
                    acc = fmaf(w[3][i], x3[i], acc);
                    acc = fmaf(w[2][i], x2[i], acc);
                    acc = fmaf(w[1][i], x1[i], acc);
                    acc = fmaf(w[0][i], x0, acc);
                    o[i] = p.silu ? zg_silu(acc) : acc;
                    x3[i] = x2[i]; x2[i] = x1[i]; x1[i] = x0;
                }
                store_vec<T, VEC>(out + (int64_t)(lb + j) * p.out_sl, o);
            }
        }
    }
}

// forward, token-major fast path: 16-bit I/O, 4 channels per thread as two fp32 pairs (zg_f2 taps), seqlen a
// multiple of CONV_LCH, everything 8-byte aligned.  ~10 issued instructions per output element instead of
// the generic kernel's 28 (ncu round 1: the generic kernel was instruction-issue bound at 52 % issue
// utilisation, 130 us for 335 MB).
template <typename T>
#ifndef ZG_CONV_PREFETCH
#define ZG_CONV_PREFETCH 0  // 1: software-pipelined row fetches (timing experiment, scripts/build_exp.sh)
#endif
#ifndef ZG_CONV_SMEM_DEFAULT
#define ZG_CONV_SMEM_DEFAULT 0      // the cp.async-staged forward kernel is opt-in until measured faster
#endif
#ifndef ZG_CONV_RCP_FMA
#define ZG_CONV_RCP_FMA 0
#endif
#ifndef ZG_CONV_MINB
#define ZG_CONV_MINB 8      // (64 registers, 8 CTAs per SM: 74.0 us vs 75.4 at 6; fetching 4 rows per batch instead of 8: 83-88 us)
#endif
__global__ void __launch_bounds__(128, ZG_CONV_MINB) conv_fwd_tok4_kernel(const zg_conv_params p) {
    static_assert(sizeof(T) == 2, "16-bit I/O");
    const int E = p.dim, L = p.seqlen, W = p.width;
    const int nvec = E >> 2;
    const int nchunk = L / CONV_LCH;
    const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (int64_t)p.batch * nchunk * nvec) return;
    const int v = (int)(gid % nvec);
    const int ch = (int)((gid / nvec) % nchunk);
    const int b = (int)(gid / ((int64_t)nvec * nchunk));
    const int e0 = v * 4;
    const int l0 = ch * CONV_LCH;
    const T *x = reinterpret_cast<const T *>(p.x) + (int64_t)b * p.x_sb + e0;
    T *out = reinterpret_cast<T *>(p.out) + (int64_t)b * p.out_sb + e0 + (int64_t)l0 * p.out_sl;
    const int xsl = (int)p.x_sl, osl = (int)p.out_sl;

    zg_f2 w[4][2], bias[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        bias[h].x = p.bias ? load_w_dt(p.bias, e0 + 2 * h, p.wdtype) : 0.f;
        bias[h].y = p.bias ? load_w_dt(p.bias, e0 + 2 * h + 1, p.wdtype) : 0.f;
#pragma unroll
        for (int k = 0; k < 4; ++k) {   // w[k] multiplies x[l - k]  (weight index W-1-k)
            w[k][h].x = (k < W) ? load_w_dt(p.weight, (int64_t)(e0 + 2 * h) * W + (W - 1 - k), p.wdtype) : 0.f;
            w[k][h].y = (k < W) ? load_w_dt(p.weight, (int64_t)(e0 + 2 * h + 1) * W + (W - 1 - k), p.wdtype) : 0.f;
        }
    }
    auto row_ptr = [&](int l) -> const uint2 * {
        const int row = p.x_rowmap ? p.x_rowmap[l] : l;
        return reinterpret_cast<const uint2 *>(x + row * xsl);
    };
    auto unpack = [](uint2 r, zg_f2 (&d)[2]) {
        if (sizeof(T) == 2 && std::is_same<T, __nv_bfloat16>::value) {
            d[0] = make_float2(__uint_as_float(r.x << 16), __uint_as_float(r.x & 0xffff0000u));
            d[1] = make_float2(__uint_as_float(r.y << 16), __uint_as_float(r.y & 0xffff0000u));
        } else {
            d[0] = __half22float2(*reinterpret_cast<const __half2 *>(&r.x));
            d[1] = __half22float2(*reinterpret_cast<const __half2 *>(&r.y));
        }
    };
    zg_f2 x1[2], x2[2], x3[2];
    const int seg = p.seg_len;      // 0, or a multiple of CONV_RB: independent segments (no taps across a segment start)
    {
        const uint2 zero = make_uint2(0u, 0u);
        const int hist = seg > 0 ? (l0 % seg) : l0;      // positions of this segment before l0
        unpack(hist >= 1 ? *row_ptr(l0 - 1) : zero, x1);
        unpack(hist >= 2 ? *row_ptr(l0 - 2) : zero, x2);
        unpack(hist >= 3 ? *row_ptr(l0 - 3) : zero, x3);
    }
#ifndef ZG_CONV_RB4
#define ZG_CONV_RB4 CONV_RB
#endif
    constexpr int RB4 = ZG_CONV_RB4;       // rows fetched per batch of independent loads in this kernel
    auto compute_batch = [&](int lb, const uint2 (&raw)[RB4]) {
        if (seg > 0 && lb > 0 && ((l0 + lb) % seg) == 0) {      // a new segment starts with this batch of rows: zero history
#pragma unroll
            for (int h = 0; h < 2; ++h) x1[h] = x2[h] = x3[h] = make_float2(0.f, 0.f);
        }
#pragma unroll
        for (int j = 0; j < RB4; ++j) {
            zg_f2 x0[2];
            unpack(raw[j], x0);
            uint2 o;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                zg_f2 acc = zg_fma2(w[3][h], x3[h], bias[h]);
                acc = zg_fma2(w[2][h], x2[h], acc);
                acc = zg_fma2(w[1][h], x1[h], acc);
                acc = zg_fma2(w[0][h], x0[h], acc);
#if ZG_CONV_RCP_FMA
                if (p.silu) {      // timing experiment (scripts/build_exp.sh): the sigmoid's reciprocal on the FMA pipe (integer seed + 3 Newton steps), 1 MUFU per value
                    float2 t = zg_mul2(acc, zg_splat2(-ZG_LOG2E));
                    t.x = fminf(t.x, 126.f); t.y = fminf(t.y, 126.f);
                    const float2 d = zg_add2(make_float2(zg_ex2(t.x), zg_ex2(t.y)), zg_splat2(1.f));
                    float2 r = make_float2(__int_as_float(0x7EF311C7 - __float_as_int(d.x)), __int_as_float(0x7EF311C7 - __float_as_int(d.y)));
                    const float2 nd = make_float2(-d.x, -d.y), one = zg_splat2(1.f);
#pragma unroll
                    for (int it = 0; it < 3; ++it) r = zg_fma2(r, zg_fma2(nd, r, one), r);
                    acc = zg_mul2(acc, r);
                }
#else
                if (p.silu) { acc.x = zg_silu(acc.x); acc.y = zg_silu(acc.y); }
#endif
                x3[h] = x2[h]; x2[h] = x1[h]; x1[h] = x0[h];
                unsigned packed;
                if (std::is_same<T, __nv_bfloat16>::value) {
                    __nv_bfloat162 t = __floats2bfloat162_rn(acc.x, acc.y);
                    packed = *reinterpret_cast<unsigned *>(&t);
                } else {
                    __half2 t = __floats2half2_rn(acc.x, acc.y);
                    packed = *reinterpret_cast<unsigned *>(&t);
                }
                if (h == 0) o.x = packed; else o.y = packed;
            }
            *reinterpret_cast<uint2 *>(out + (lb + j) * osl) = o;
        }
    };
#if ZG_CONV_PREFETCH
    // software-pipelined: the rows of batch k + 1 are in flight while batch k is computed (ncu of the plain loop: long_scoreboard
    // 5.4 warps per issue -- every warp waits for its own batch before it computes anything)
    static_assert((CONV_LCH / RB4) % 2 == 0, "an even number of batches");
    uint2 ra[RB4], rb[RB4];
#pragma unroll
    for (int j = 0; j < RB4; ++j) ra[j] = *row_ptr(l0 + j);
#pragma unroll 1
    for (int lb = 0; lb < CONV_LCH; lb += 2 * RB4) {
#pragma unroll
        for (int j = 0; j < RB4; ++j) rb[j] = *row_ptr(l0 + lb + RB4 + j);
        compute_batch(lb, ra);
        if (lb + 2 * RB4 < CONV_LCH) {
#pragma unroll
            for (int j = 0; j < RB4; ++j) ra[j] = *row_ptr(l0 + lb + 2 * RB4 + j);
        }
        compute_batch(lb + RB4, rb);
    }
#else
#pragma unroll 1
    for (int lb = 0; lb < CONV_LCH; lb += RB4) {
        uint2 raw[RB4];
#pragma unroll
        for (int j = 0; j < RB4; ++j) raw[j] = *row_ptr(l0 + lb + j);
        compute_batch(lb, raw);
    }
#endif
}

// forward, token-major, rows staged through shared memory by cp.async (opt-in: ZG_CONV_SMEM=1).
// Why: ncu of conv_fwd_tok4_kernel shows a latency-bound kernel (long_scoreboard 5.4 warps per issue at 0.69 of the HBM roofline): a
// thread has its 8 rows x 8 bytes in flight only while it is NOT computing, and registers for a second batch cost more occupancy than
// the prefetch hides (ZG_CONV_PREFETCH, rejected).  Here a lane owns 8 adjacent channels (16 bytes per row) and keeps TWO batches of 8
// rows in flight in a per-lane shared-memory ring (3 batches x 8 rows x 16 B) while it computes the third: 128 KB in flight per SM with
// 16 resident warps, no registers spent on data in flight.  Every lane reads back exactly the 16 bytes it copied itself, so its own
// cp.async.wait_group is the only synchronisation (no barrier, no __syncwarp).  Same arithmetic and rounding as conv_fwd_tok4_kernel
// (zg_f2 taps in the same order, the same SiLU): bit-identical results.
constexpr int CS_ROWS = 8, CS_STAGES = 3, CS_WARPS = 4, CS_CH = 256;          // rows per batch, ring depth, warps per CTA, channels per warp
constexpr int CS_WARP_BYTES = CS_STAGES * CS_ROWS * CS_CH * 2;                // 12 KB
template <typename T, int LCH>
__global__ void __launch_bounds__(32 * CS_WARPS, 4) conv_fwd_tok8s_kernel(const zg_conv_params p) {
    static_assert(sizeof(T) == 2, "16-bit I/O");
    static_assert(LCH % CS_ROWS == 0 && LCH / CS_ROWS >= 2, "whole batches");
    extern __shared__ __align__(16) unsigned char conv_smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int E = p.dim, L = p.seqlen, W = p.width;
    const int nv = E / CS_CH, nchunk = L / LCH;
    const int64_t wid = (int64_t)blockIdx.x * CS_WARPS + warp;
    if (wid >= (int64_t)p.batch * nchunk * nv) return;          // (no block-wide barrier anywhere below)
    const int v = (int)(wid % nv);
    const int ch = (int)((wid / nv) % nchunk);
    const int b = (int)(wid / ((int64_t)nv * nchunk));
    const int e0 = v * CS_CH + lane * 8;
    const int l0 = ch * LCH;
    const T *x = reinterpret_cast<const T *>(p.x) + (int64_t)b * p.x_sb + e0;
    T *out = reinterpret_cast<T *>(p.out) + (int64_t)b * p.out_sb + e0 + (int64_t)l0 * p.out_sl;
    const int xsl = (int)p.x_sl, osl = (int)p.out_sl;
    unsigned char *ring = conv_smem + warp * CS_WARP_BYTES + lane * 16;      // this lane's 16 bytes of row r of batch slot s: + (s * CS_ROWS + r) * 512

    zg_f2 w[4][4], bias[4];
#pragma unroll
    for (int h = 0; h < 4; ++h) {
        bias[h].x = p.bias ? load_w_dt(p.bias, e0 + 2 * h, p.wdtype) : 0.f;
        bias[h].y = p.bias ? load_w_dt(p.bias, e0 + 2 * h + 1, p.wdtype) : 0.f;
#pragma unroll
        for (int k = 0; k < 4; ++k) {   // w[k] multiplies x[l - k]  (weight index W-1-k)
            w[k][h].x = (k < W) ? load_w_dt(p.weight, (int64_t)(e0 + 2 * h) * W + (W - 1 - k), p.wdtype) : 0.f;
            w[k][h].y = (k < W) ? load_w_dt(p.weight, (int64_t)(e0 + 2 * h + 1) * W + (W - 1 - k), p.wdtype) : 0.f;
        }
    }
    auto row_ptr = [&](int l) -> const unsigned char * {
        const int row = p.x_rowmap ? p.x_rowmap[l] : l;
        return reinterpret_cast<const unsigned char *>(x + row * xsl);
    };
    auto unpack = [](uint4 r, zg_f2 (&d)[4]) {
        const unsigned rr[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
        for (int h = 0; h < 4; ++h) {
            if (std::is_same<T, __nv_bfloat16>::value) d[h] = make_float2(__uint_as_float(rr[h] << 16), __uint_as_float(rr[h] & 0xffff0000u));
            else d[h] = __half22float2(*reinterpret_cast<const __half2 *>(&rr[h]));
        }
    };
    constexpr int NB = LCH / CS_ROWS;
    auto issue = [&](int k) {           // the 8 rows of batch k -> ring slot k % CS_STAGES, one commit group
        unsigned char *dst = ring + (k % CS_STAGES) * (CS_ROWS * CS_CH * 2);
#pragma unroll
        for (int j = 0; j < CS_ROWS; ++j) zg_cp_async16(dst + j * (CS_CH * 2), row_ptr(l0 + k * CS_ROWS + j));
        zg_cp_async_commit();
    };
    issue(0);
    issue(1);
    zg_f2 x1[4], x2[4], x3[4];
    const int seg = p.seg_len;      // 0, or a multiple of CS_ROWS: independent segments (no taps across a segment start)
    {
        const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
        const int hist = seg > 0 ? (l0 % seg) : l0;      // positions of this segment before l0
        unpack(hist >= 1 ? *reinterpret_cast<const uint4 *>(row_ptr(l0 - 1)) : zero, x1);
        unpack(hist >= 2 ? *reinterpret_cast<const uint4 *>(row_ptr(l0 - 2)) : zero, x2);
        unpack(hist >= 3 ? *reinterpret_cast<const uint4 *>(row_ptr(l0 - 3)) : zero, x3);
    }
#pragma unroll 1
    for (int k = 0; k < NB; ++k) {
        if (k + 2 < NB) issue(k + 2);           // slot (k - 1) % 3: its rows were consumed (and stored) in the previous iteration
        else zg_cp_async_commit();              // empty group: the wait below always leaves exactly two groups pending
        zg_cp_async_wait<2>();                  // this lane's copies of batch k have landed
        const int lb = k * CS_ROWS;
        if (seg > 0 && lb > 0 && ((l0 + lb) % seg) == 0) {      // a new segment starts with this batch of rows: zero history
#pragma unroll
            for (int h = 0; h < 4; ++h) x1[h] = x2[h] = x3[h] = make_float2(0.f, 0.f);
        }
        const unsigned char *src = ring + (k % CS_STAGES) * (CS_ROWS * CS_CH * 2);
#pragma unroll
        for (int j = 0; j < CS_ROWS; ++j) {
            zg_f2 x0[4];
            unpack(*reinterpret_cast<const uint4 *>(src + j * (CS_CH * 2)), x0);
            unsigned o[4];
#pragma unroll
            for (int h = 0; h < 4; ++h) {
                zg_f2 acc = zg_fma2(w[3][h], x3[h], bias[h]);
                acc = zg_fma2(w[2][h], x2[h], acc);
                acc = zg_fma2(w[1][h], x1[h], acc);
                acc = zg_fma2(w[0][h], x0[h], acc);
                if (p.silu) { acc.x = zg_silu(acc.x); acc.y = zg_silu(acc.y); }
                x3[h] = x2[h]; x2[h] = x1[h]; x1[h] = x0[h];
                if (std::is_same<T, __nv_bfloat16>::value) {
                    __nv_bfloat162 t = __floats2bfloat162_rn(acc.x, acc.y);
                    o[h] = *reinterpret_cast<unsigned *>(&t);
                } else {
                    __half2 t = __floats2half2_rn(acc.x, acc.y);
                    o[h] = *reinterpret_cast<unsigned *>(&t);
                }
            }
            *reinterpret_cast<uint4 *>(out + (lb + j) * osl) = make_uint4(o[0], o[1], o[2], o[3]);
        }
    }
}

// forward, seq-contiguous
template <typename T, int VEC>
__global__ void __launch_bounds__(128) conv_fwd_seqc_kernel(const zg_conv_params p) {
    const int E = p.dim, L = p.seqlen, W = p.width;
    const int nvec = (L + VEC - 1) / VEC;
    const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (int64_t)p.batch * E * nvec) return;
    const int v = (int)(gid % nvec);
    const int e = (int)((gid / nvec) % E);
    const int b = (int)(gid / ((int64_t)nvec * E));
    const int l0 = v * VEC;
    const T *x = reinterpret_cast<const T *>(p.x) + (int64_t)b * p.x_sb + (int64_t)e * p.x_sd;
    T *out = reinterpret_cast<T *>(p.out) + (int64_t)b * p.out_sb + (int64_t)e * p.out_sd;
    float w[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) w[k] = k < W ? load_w_dt(p.weight, (int64_t)e * W + (W - 1 - k), p.wdtype) : 0.f;
    const float bias = p.bias ? load_w_dt(p.bias, e, p.wdtype) : 0.f;
    float win[VEC + 3];   // win[3 + i] = x[l0 + i]
    if (VEC > 1) {
        float cur[VEC], prev[VEC];
        load_vec<T, VEC>(cur, x + l0);
        if (l0 > 0) load_vec<T, VEC>(prev, x + l0 - VEC);
#pragma unroll
        for (int i = 0; i < VEC; ++i) win[3 + i] = cur[i];
#pragma unroll
        for (int i = 0; i < 3; ++i) win[i] = (l0 > 0) ? prev[VEC - 3 + i] : 0.f;
    } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) win[i] = (l0 - 3 + i >= 0) ? zg_to_float<T>(x[l0 - 3 + i]) : 0.f;
    }
    float o[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
        float acc = bias;
        acc = fmaf(w[3], win[i], acc);
        acc = fmaf(w[2], win[i + 1], acc);
        acc = fmaf(w[1], win[i + 2], acc);
        acc = fmaf(w[0], win[i + 3], acc);
        o[i] = p.silu ? zg_silu(acc) : acc;
    }
    store_vec<T, VEC>(out + l0, o);
}

// ------------------------------------------------------------------------------------------------
// backward, seq-contiguous (the autograd path of causal_conv1d_fn; causal_conv1d_bwd.cu:46-240).
// One warp per (batch, channel) row: lanes stride over l, dx written, dweight/dbias reduced in the
// warp and accumulated with one fp32 atomicAdd per (row, tap).
//   g[l]   = dout[l] * (silu ? silu'(pre[l]) : 1),  pre[l] = bias + sum_k w[k] x[l-k]
//   dx[l]  = sum_k w[k] g[l+k]          dw[k] = sum_l g[l] x[l-k]        db = sum_l g[l]
// DET (both channel-first kernels): dweight / dbias of q address partial rows, one per batch row -- (batch, dim, width) /
// (batch, dim) -- stored, not added (zg_causal_conv1d_bwd_det).
template <typename T, bool DET>
__global__ void __launch_bounds__(128) conv_bwd_seqc_kernel(const zg_conv_bwd_params q) {
    const zg_conv_params &p = q.fwd;
    const int E = p.dim, L = p.seqlen, W = p.width;
    const int warp = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (warp >= p.batch * E) return;
    const int b = warp / E, e = warp % E;
    const T *x = reinterpret_cast<const T *>(p.x) + (int64_t)b * p.x_sb + (int64_t)e * p.x_sd;
    const T *dout = reinterpret_cast<const T *>(q.dout) + (int64_t)b * q.dout_sb + (int64_t)e * q.dout_sd;
    T *dx = reinterpret_cast<T *>(q.dx) + (int64_t)b * q.dx_sb + (int64_t)e * q.dx_sd;
    float w[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) w[k] = k < W ? load_w_dt(p.weight, (int64_t)e * W + (W - 1 - k), p.wdtype) : 0.f;
    const float bias = p.bias ? load_w_dt(p.bias, e, p.wdtype) : 0.f;
    auto X = [&](int l) { return (l >= 0 && l < L) ? zg_to_float<T>(x[l]) : 0.f; };
    auto G = [&](int l) {   // gradient wrt the pre-activation at position l
        if (l < 0 || l >= L) return 0.f;
        float g = zg_to_float<T>(dout[l]);
        if (p.silu) {
            const float pre = bias + w[0] * X(l) + w[1] * X(l - 1) + w[2] * X(l - 2) + w[3] * X(l - 3);
            const float s = 1.f / (1.f + __expf(-pre));
            g *= s * (1.f + pre * (1.f - s));
        }
        return g;
    };
    float dw[4] = {0.f, 0.f, 0.f, 0.f}, db = 0.f;
    for (int l = lane; l < L; l += 32) {
        const float g0 = G(l), g1 = G(l + 1), g2 = G(l + 2), g3 = G(l + 3);
        dx[l] = zg_from_float<T>(w[0] * g0 + w[1] * g1 + w[2] * g2 + w[3] * g3);
        db += g0;
#pragma unroll
        for (int k = 0; k < 4; ++k) dw[k] += g0 * X(l - k);
    }
    db = zg_warp_sum(db);
#pragma unroll
    for (int k = 0; k < 4; ++k) dw[k] = zg_warp_sum(dw[k]);
    if (DET && lane == 0) {
        const int64_t be = (int64_t)b * E + e;
        if (q.dbias) q.dbias[be] = db;
        for (int k = 0; k < W; ++k) q.dweight[be * W + (W - 1 - k)] = dw[k];
    } else if (lane == 0) {
        if (q.dbias) atomicAdd(q.dbias + e, db);
        for (int k = 0; k < W; ++k) atomicAdd(q.dweight + (int64_t)e * W + (W - 1 - k), dw[k]);
    }
}


// backward, seq-contiguous (channel-first), vector path: one warp per (batch, channel) row; a lane owns VEC
// consecutive positions of a 32 * VEC tile (one 16-byte load of x and of dout, one 16-byte store of dx), the
// x halo comes from the lane below and the g halo from the lane above by shuffles; tiles are walked from the
// END of the row so that the three g values the last lane needs from the next tile are already known.  Each
// silu' is evaluated once (the scalar kernel above evaluates it four times per position).
template <typename T, bool DET>
__global__ void __launch_bounds__(128) conv_bwd_seqc_vec_kernel(const zg_conv_bwd_params q) {
    constexpr int VEC = 16 / (int)sizeof(T);
    const zg_conv_params &p = q.fwd;
    const int E = p.dim, L = p.seqlen, W = p.width;
    const int warp = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (warp >= p.batch * E) return;
    const int b = warp / E, e = warp % E;
    const T *x = reinterpret_cast<const T *>(p.x) + (int64_t)b * p.x_sb + (int64_t)e * p.x_sd;
    const T *dout = reinterpret_cast<const T *>(q.dout) + (int64_t)b * q.dout_sb + (int64_t)e * q.dout_sd;
    T *dx = reinterpret_cast<T *>(q.dx) + (int64_t)b * q.dx_sb + (int64_t)e * q.dx_sd;
    float w[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) w[k] = k < W ? load_w_dt(p.weight, (int64_t)e * W + (W - 1 - k), p.wdtype) : 0.f;
    const float bias = p.bias ? load_w_dt(p.bias, e, p.wdtype) : 0.f;
    float dw[4] = {0.f, 0.f, 0.f, 0.f}, db = 0.f;
    float gn[3] = {0.f, 0.f, 0.f};                 // g at the first three positions of the tile above (0 past the end)
    const int ntiles = (L + 32 * VEC - 1) / (32 * VEC);
    for (int tile = ntiles - 1; tile >= 0; --tile) {
        const int l = tile * 32 * VEC + lane * VEC;          // first position of this lane (L % VEC == 0: all-or-nothing)
        const bool in = l < L;
        float xv[VEC + 3], g[VEC + 3];                        // xv[j] = x[l - 3 + j];  g[j] = g[l + j]
        float go[VEC];
        if (in) {
            load_vec<T, VEC>(*reinterpret_cast<float(*)[VEC]>(&xv[3]), x + l);
            load_vec<T, VEC>(go, dout + l);
        } else {
#pragma unroll
            for (int j = 0; j < VEC; ++j) { xv[3 + j] = 0.f; go[j] = 0.f; }
        }
        // x halo: the last three positions of the lane below; lane 0 reads them from memory
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const float up = __shfl_up_sync(0xffffffffu, xv[VEC + j], 1);
            xv[j] = up;
        }
        if (lane == 0) {
#pragma unroll
            for (int j = 0; j < 3; ++j) xv[j] = (l - 3 + j >= 0 && in) ? zg_to_float<T>(x[l - 3 + j]) : 0.f;
        }
#pragma unroll
        for (int j = 0; j < VEC; ++j) {
            float gg = go[j];
            if (p.silu) {
                const float pre = fmaf(w[0], xv[j + 3], fmaf(w[1], xv[j + 2], fmaf(w[2], xv[j + 1], fmaf(w[3], xv[j], bias))));
                const float sg = zg_sigmoid(pre);
                gg *= sg * fmaf(pre, 1.f - sg, 1.f);
            }
            g[j] = in ? gg : 0.f;
            db += g[j];
            dw[0] = fmaf(g[j], xv[j + 3], dw[0]);
            dw[1] = fmaf(g[j], xv[j + 2], dw[1]);
            dw[2] = fmaf(g[j], xv[j + 1], dw[2]);
            dw[3] = fmaf(g[j], xv[j], dw[3]);
        }
        // g halo: the first three positions of the lane above; the last lane takes the tile above's
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const float dn = __shfl_down_sync(0xffffffffu, g[j], 1);
            g[VEC + j] = (lane == 31) ? gn[j] : dn;
        }
        if (in) {
            float o[VEC];
#pragma unroll
            for (int j = 0; j < VEC; ++j) o[j] = fmaf(w[0], g[j], fmaf(w[1], g[j + 1], fmaf(w[2], g[j + 2], w[3] * g[j + 3])));
            store_vec<T, VEC>(dx + l, o);
        }
#pragma unroll
        for (int j = 0; j < 3; ++j) gn[j] = __shfl_sync(0xffffffffu, g[j], 0);
    }
    db = zg_warp_sum(db);
#pragma unroll
    for (int k = 0; k < 4; ++k) dw[k] = zg_warp_sum(dw[k]);
    if (DET && lane == 0) {
        const int64_t be = (int64_t)b * E + e;
        if (q.dbias) q.dbias[be] = db;
        for (int k = 0; k < W; ++k) q.dweight[be * W + (W - 1 - k)] = dw[k];
    } else if (lane == 0) {
        if (q.dbias) atomicAdd(q.dbias + e, db);
        for (int k = 0; k < W; ++k) atomicAdd(q.dweight + (int64_t)e * W + (W - 1 - k), dw[k]);
    }
}

// backward, dim-contiguous (token-major): a thread owns DV adjacent channels and CONV_BLCH consecutive
// positions and streams upwards in l with two sliding windows (x[l-3..l] for the pre-activation,
// g[l-3..l] for dx[l-3] = sum_k w[k] g[l-3+k]); the three positions after the chunk are walked as a
// halo (their g feeds the chunk's last dx, their dw/db belong to the next chunk).  x_rowmap[l]
// redirects both the x reads and the dx writes (the conv ran over the permuted sequence; dx goes
// back to token order).  dweight/dbias: summed over the 4 warps of the CTA (4 chunks of the same
// channels) in shared memory, then one atomic per (CTA, channel, tap).
// DET (both token-major kernels): dweight / dbias of q address partial rows, one per CTA row group blockIdx.x / nvb
// (= 4 consecutive (batch, chunk) rows) -- (ceil(batch * nchunk / 4), dim, width) / (.., dim) -- stored, not added.
constexpr int CONV_BLCH = 64;
constexpr int CONV_BRB = 4;     // rows per batch of independent loads in the backward (x and dout: 2 * CONV_BRB loads in flight)

template <typename T, int DV, int BRB, bool DET>
__global__ void __launch_bounds__(128, (DV <= 2) ? 6 : 4) conv_bwd_tok_kernel(const zg_conv_bwd_params q) {
    const zg_conv_params &p = q.fwd;
    const int E = p.dim, L = p.seqlen, W = p.width;
    const int nvec = E / DV;
    const int nvb = (nvec + 31) >> 5;
    const int nchunk = (L + CONV_BLCH - 1) / CONV_BLCH;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int v = (int)(blockIdx.x % nvb) * 32 + lane;
    const int64_t row = (int64_t)(blockIdx.x / nvb) * 4 + warp;          // enumerates (batch, chunk)
    const bool live = v < nvec && row < (int64_t)p.batch * nchunk;
    __shared__ float red[4][5 * DV][32];

    float dw[4][DV], db[DV];
#pragma unroll
    for (int i = 0; i < DV; ++i) {
        db[i] = 0.f;
#pragma unroll
        for (int k = 0; k < 4; ++k) dw[k][i] = 0.f;
    }
    const int e0 = v * DV;
    if (live) {
        const int b = (int)(row / nchunk), l0 = (int)(row % nchunk) * CONV_BLCH;
        const T *x = reinterpret_cast<const T *>(p.x) + (int64_t)b * p.x_sb + e0;
        const T *dout = reinterpret_cast<const T *>(q.dout) + (int64_t)b * q.dout_sb + e0;
        T *dx = reinterpret_cast<T *>(q.dx) + (int64_t)b * q.dx_sb + e0;
        float w[4][DV], bias[DV];
#pragma unroll
        for (int i = 0; i < DV; ++i) {
            bias[i] = p.bias ? load_w_dt(p.bias, e0 + i, p.wdtype) : 0.f;
#pragma unroll
            for (int k = 0; k < 4; ++k) w[k][i] = (k < W) ? load_w_dt(p.weight, (int64_t)(e0 + i) * W + (W - 1 - k), p.wdtype) : 0.f;
        }
        auto rowof = [&](int l) -> int64_t { return p.x_rowmap ? p.x_rowmap[l] : l; };
        float x1[DV], x2[DV], x3[DV], g1[DV], g2[DV], g3[DV];
#pragma unroll
        for (int i = 0; i < DV; ++i) { x1[i] = x2[i] = x3[i] = 0.f; g1[i] = g2[i] = g3[i] = 0.f; }
        // x window before the chunk; g window: positions l0-1.. are only needed for dx of the PREVIOUS chunk
        if (l0 >= 1) load_vec<T, DV>(x1, x + rowof(l0 - 1) * p.x_sl);
        if (l0 >= 2) load_vec<T, DV>(x2, x + rowof(l0 - 2) * p.x_sl);
        if (l0 >= 3) load_vec<T, DV>(x3, x + rowof(l0 - 3) * p.x_sl);
        const int lend = min(l0 + CONV_BLCH, L);
        const int lhalo = min(lend + 3, L);
        // positions are walked in batches of BRB rows, software pipelined: the 2 * BRB row loads of batch k + 1 are issued
        // before batch k is consumed (a thread's batches are sequential; without the prefetch every batch paid a full
        // HBM round trip: 60 us per 64-position chunk, ncu round 1)
        VecT<T, DV> xr[BRB], gr[BRB], xn[BRB], gn[BRB];
        auto fetch = [&](int lb, VecT<T, DV> (&xd)[BRB], VecT<T, DV> (&gd)[BRB]) {
#pragma unroll
            for (int j = 0; j < BRB; ++j) {
                const int l = lb + j;
                if (l < lhalo) {
                    xd[j] = *reinterpret_cast<const VecT<T, DV> *>(x + rowof(l) * p.x_sl);
                    gd[j] = *reinterpret_cast<const VecT<T, DV> *>(dout + (int64_t)l * q.dout_sl);
                }
            }
        };
        fetch(l0, xr, gr);
#pragma unroll 1
        for (int lb = l0; lb < lend + 3; lb += BRB) {
            if (lb + BRB < lend + 3) fetch(lb + BRB, xn, gn);
#pragma unroll
            for (int j = 0; j < BRB; ++j) {
                const int l = lb + j;
                float g0[DV], x0[DV];
                if (l < lhalo) {
#pragma unroll
                    for (int i = 0; i < DV; ++i) {
                        x0[i] = zg_to_float<T>(xr[j].e[i]);
                        float gg = zg_to_float<T>(gr[j].e[i]);
                        if (p.silu) {
                            const float pre = fmaf(w[0][i], x0[i], fmaf(w[1][i], x1[i], fmaf(w[2][i], x2[i], fmaf(w[3][i], x3[i], bias[i]))));
                            const float sg = zg_sigmoid(pre);
                            gg *= sg * fmaf(pre, 1.f - sg, 1.f);
                        }
                        g0[i] = gg;
                    }
                    if (l < lend) {
#pragma unroll
                        for (int i = 0; i < DV; ++i) {
                            db[i] += g0[i];
                            dw[0][i] = fmaf(g0[i], x0[i], dw[0][i]);
                            dw[1][i] = fmaf(g0[i], x1[i], dw[1][i]);
                            dw[2][i] = fmaf(g0[i], x2[i], dw[2][i]);
                            dw[3][i] = fmaf(g0[i], x3[i], dw[3][i]);
                        }
                    }
                } else {
#pragma unroll
                    for (int i = 0; i < DV; ++i) { g0[i] = 0.f; x0[i] = 0.f; }
                }
                const int m = l - 3;                      // dx[m] = w0 g[m] + w1 g[m+1] + w2 g[m+2] + w3 g[m+3]
                if (m >= l0 && m < lend) {
                    float o[DV];
#pragma unroll
                    for (int i = 0; i < DV; ++i) o[i] = fmaf(w[0][i], g3[i], fmaf(w[1][i], g2[i], fmaf(w[2][i], g1[i], w[3][i] * g0[i])));
                    store_vec<T, DV>(dx + rowof(m) * q.dx_sl, o);
                }
#pragma unroll
                for (int i = 0; i < DV; ++i) { x3[i] = x2[i]; x2[i] = x1[i]; x1[i] = x0[i]; g3[i] = g2[i]; g2[i] = g1[i]; g1[i] = g0[i]; }
            }
#pragma unroll
            for (int j = 0; j < BRB; ++j) { xr[j] = xn[j]; gr[j] = gn[j]; }
        }
    }
    // CTA reduction of the weight / bias gradients over the 4 warps
#pragma unroll
    for (int i = 0; i < DV; ++i) {
        red[warp][4 * DV + i][lane] = db[i];
#pragma unroll
        for (int k = 0; k < 4; ++k) red[warp][k * DV + i][lane] = dw[k][i];
    }
    __syncthreads();
    for (int it = threadIdx.x; it < 5 * DV * 32; it += 128) {
        const int j = it >> 5, ln = it & 31;
        const int vv = (int)(blockIdx.x % nvb) * 32 + ln;
        if (vv >= nvec) continue;
        const float sum = red[0][j][ln] + red[1][j][ln] + red[2][j][ln] + red[3][j][ln];
        const int k = j / DV, i = j % DV, e = vv * DV + i;
        if constexpr (DET) {
            const int64_t re = (int64_t)(blockIdx.x / nvb) * E + e;
            if (k == 4) { if (q.dbias) q.dbias[re] = sum; }
            else if (k < W) q.dweight[re * W + (W - 1 - k)] = sum;
        } else {
            if (k == 4) { if (q.dbias) atomicAdd(q.dbias + e, sum); }
            else if (k < W) atomicAdd(q.dweight + (int64_t)e * W + (W - 1 - k), sum);
        }
    }
}

// backward, token-major FAST path (16-bit I/O, dim % 4 == 0, seqlen % CONV_B4_LCH == 0, aligned): same streaming scheme
// as conv_bwd_tok_kernel but branch-free -- chunks are whole, the three halo positions either all exist (another chunk
// follows) or none does, so the per-position bounds tests, the divergent branches and most of the address arithmetic of
// the generic kernel go away (ncu round 1: 66 issued instructions per channel-position there, ~25 needed), rows are
// fetched CONV_B4_RB at a time one batch ahead, taps run as zg_f2 FMAs on channel pairs.
constexpr int CONV_B4_LCH = 32;
constexpr int CONV_B4_RB = 4;

template <typename T, bool HAS_MAP, bool DET>
__global__ void __launch_bounds__(128, 4) conv_bwd_tok4_kernel(const zg_conv_bwd_params q) {
    static_assert(sizeof(T) == 2, "16-bit I/O");
    constexpr int LCH = CONV_B4_LCH, RB = CONV_B4_RB;
    const zg_conv_params &p = q.fwd;
    const int E = p.dim, L = p.seqlen, W = p.width;
    const int nvec = E >> 2;
    const int nvb = (nvec + 31) >> 5;
    const int nchunk = L / LCH;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int v = (int)(blockIdx.x % nvb) * 32 + lane;
    const int64_t row = (int64_t)(blockIdx.x / nvb) * 4 + warp;          // enumerates (batch, chunk)
    const bool live = v < nvec && row < (int64_t)p.batch * nchunk;
    __shared__ float red[4][20][32];
    zg_f2 dw[4][2], db[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        db[h] = zg_splat2(0.f);
#pragma unroll
        for (int k = 0; k < 4; ++k) dw[k][h] = zg_splat2(0.f);
    }
    const int e0 = v * 4;
    if (live) {
        const int b = (int)(row / nchunk), l0 = (int)(row % nchunk) * LCH;
        const bool halo = l0 + LCH < L;
        const T *x = reinterpret_cast<const T *>(p.x) + (int64_t)b * p.x_sb + e0;
        const T *dout = reinterpret_cast<const T *>(q.dout) + (int64_t)b * q.dout_sb + e0;
        T *dx = reinterpret_cast<T *>(q.dx) + (int64_t)b * q.dx_sb + e0;
        const int xsl = (int)p.x_sl, gsl = (int)q.dout_sl, dsl = (int)q.dx_sl;
        const int32_t *rm = p.x_rowmap;
        zg_f2 w[4][2], bias[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            bias[h].x = p.bias ? load_w_dt(p.bias, e0 + 2 * h, p.wdtype) : 0.f;
            bias[h].y = p.bias ? load_w_dt(p.bias, e0 + 2 * h + 1, p.wdtype) : 0.f;
#pragma unroll
            for (int k = 0; k < 4; ++k) {   // w[k] multiplies x[l - k]
                w[k][h].x = (k < W) ? load_w_dt(p.weight, (int64_t)(e0 + 2 * h) * W + (W - 1 - k), p.wdtype) : 0.f;
                w[k][h].y = (k < W) ? load_w_dt(p.weight, (int64_t)(e0 + 2 * h + 1) * W + (W - 1 - k), p.wdtype) : 0.f;
            }
        }
        auto xrow = [&](int l) -> const uint2 * { return reinterpret_cast<const uint2 *>(x + (HAS_MAP ? rm[l] : l) * xsl); };
        auto unpack = [](uint2 r, zg_f2 (&d)[2]) {
            if (std::is_same<T, __nv_bfloat16>::value) {
                d[0] = make_float2(__uint_as_float(r.x << 16), __uint_as_float(r.x & 0xffff0000u));
                d[1] = make_float2(__uint_as_float(r.y << 16), __uint_as_float(r.y & 0xffff0000u));
            } else {
                d[0] = __half22float2(*reinterpret_cast<const __half2 *>(&r.x));
                d[1] = __half22float2(*reinterpret_cast<const __half2 *>(&r.y));
            }
        };
        auto pack = [](const zg_f2 (&o)[2]) -> uint2 {
            uint2 r;
            if (std::is_same<T, __nv_bfloat16>::value) {
                __nv_bfloat162 a = __floats2bfloat162_rn(o[0].x, o[0].y), c = __floats2bfloat162_rn(o[1].x, o[1].y);
                r.x = *reinterpret_cast<unsigned *>(&a); r.y = *reinterpret_cast<unsigned *>(&c);
            } else {
                __half2 a = __floats2half2_rn(o[0].x, o[0].y), c = __floats2half2_rn(o[1].x, o[1].y);
                r.x = *reinterpret_cast<unsigned *>(&a); r.y = *reinterpret_cast<unsigned *>(&c);
            }
            return r;
        };
        zg_f2 x1[2], x2[2], x3[2], g1[2], g2[2], g3[2];
        const uint2 zero = make_uint2(0u, 0u);
        unpack(l0 >= 1 ? *xrow(l0 - 1) : zero, x1);
        unpack(l0 >= 2 ? *xrow(l0 - 2) : zero, x2);
        unpack(l0 >= 3 ? *xrow(l0 - 3) : zero, x3);
#pragma unroll
        for (int h = 0; h < 2; ++h) g1[h] = g2[h] = g3[h] = zg_splat2(0.f);
        // one position: pre-activation, g = dout * silu'(pre), weight-gradient taps, dx of the position three back
        auto step = [&](uint2 rawx, uint2 rawg, bool acc, bool emit, int m) {
            zg_f2 x0[2], g0[2], o[2];
            unpack(rawx, x0);
            unpack(rawg, g0);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (p.silu) {
                    zg_f2 pre = zg_fma2(w[3][h], x3[h], bias[h]);
                    pre = zg_fma2(w[2][h], x2[h], pre);
                    pre = zg_fma2(w[1][h], x1[h], pre);
                    pre = zg_fma2(w[0][h], x0[h], pre);
                    const zg_f2 sg = make_float2(zg_sigmoid(pre.x), zg_sigmoid(pre.y));
                    const zg_f2 one = zg_splat2(1.f);
                    // silu'(pre) = sg * (1 + pre * (1 - sg))
                    const zg_f2 t = zg_fma2(pre, zg_fma2(sg, zg_splat2(-1.f), one), one);
                    g0[h] = zg_mul2(g0[h], zg_mul2(sg, t));
                }
                if (acc) {
                    db[h] = zg_add2(db[h], g0[h]);
                    dw[0][h] = zg_fma2(g0[h], x0[h], dw[0][h]);
                    dw[1][h] = zg_fma2(g0[h], x1[h], dw[1][h]);
                    dw[2][h] = zg_fma2(g0[h], x2[h], dw[2][h]);
                    dw[3][h] = zg_fma2(g0[h], x3[h], dw[3][h]);
                }
                o[h] = zg_fma2(w[0][h], g3[h], zg_fma2(w[1][h], g2[h], zg_fma2(w[2][h], g1[h], zg_mul2(w[3][h], g0[h]))));
                x3[h] = x2[h]; x2[h] = x1[h]; x1[h] = x0[h]; g3[h] = g2[h]; g2[h] = g1[h]; g1[h] = g0[h];
            }
            if (emit) *reinterpret_cast<uint2 *>(dx + (HAS_MAP ? rm[m] : m) * dsl) = pack(o);
        };
        uint2 cx[RB], cg[RB], nx[RB], ng[RB];
#pragma unroll
        for (int j = 0; j < RB; ++j) { cx[j] = *xrow(l0 + j); cg[j] = *reinterpret_cast<const uint2 *>(dout + (l0 + j) * gsl); }
#pragma unroll 1
        for (int lb = l0; lb < l0 + LCH; lb += RB) {
            const bool more = lb + RB < l0 + LCH;
            if (more) {
#pragma unroll
                for (int j = 0; j < RB; ++j) { nx[j] = *xrow(lb + RB + j); ng[j] = *reinterpret_cast<const uint2 *>(dout + (lb + RB + j) * gsl); }
            } else if (halo) {
#pragma unroll
                for (int j = 0; j < 3; ++j) { nx[j] = *xrow(lb + RB + j); ng[j] = *reinterpret_cast<const uint2 *>(dout + (lb + RB + j) * gsl); }
            }
#pragma unroll
            for (int j = 0; j < RB; ++j) step(cx[j], cg[j], true, lb + j - 3 >= l0, lb + j - 3);
#pragma unroll
            for (int j = 0; j < RB; ++j) { cx[j] = nx[j]; cg[j] = ng[j]; }
        }
        // the three positions after the chunk: they only feed the chunk's last three dx
#pragma unroll
        for (int j = 0; j < 3; ++j) step(halo ? cx[j] : zero, halo ? cg[j] : zero, false, true, l0 + LCH - 3 + j);
    }
    // CTA reduction of the weight / bias gradients over the 4 warps (4 chunks of the same channels)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        red[warp][16 + 2 * h][lane] = db[h].x; red[warp][16 + 2 * h + 1][lane] = db[h].y;
#pragma unroll
        for (int k = 0; k < 4; ++k) { red[warp][k * 4 + 2 * h][lane] = dw[k][h].x; red[warp][k * 4 + 2 * h + 1][lane] = dw[k][h].y; }
    }
    __syncthreads();
    for (int it = threadIdx.x; it < 20 * 32; it += 128) {
        const int j = it >> 5, ln = it & 31;
        const int vv = (int)(blockIdx.x % nvb) * 32 + ln;
        if (vv >= nvec) continue;
        const float sum = red[0][j][ln] + red[1][j][ln] + red[2][j][ln] + red[3][j][ln];
        const int k = j >> 2, i = j & 3, e = vv * 4 + i;
        if constexpr (DET) {
            const int64_t re = (int64_t)(blockIdx.x / nvb) * E + e;
            if (k == 4) { if (q.dbias) q.dbias[re] = sum; }
            else if (k < W) q.dweight[re * W + (W - 1 - k)] = sum;
        } else {
            if (k == 4) { if (q.dbias) atomicAdd(q.dbias + e, sum); }
            else if (k < W) atomicAdd(q.dweight + (int64_t)e * W + (W - 1 - k), sum);
        }
    }
}

template <typename T> static int conv_fwd_t(const zg_conv_params &p, bool seq, cudaStream_t s) {
    constexpr int VEC = 16 / sizeof(T);
    const uintptr_t align_bits = reinterpret_cast<uintptr_t>(p.x) | reinterpret_cast<uintptr_t>(p.out);
    if (seq) {
        const bool vec_ok = (p.seqlen % VEC == 0) && (align_bits % 16 == 0) && (p.x_sb % VEC == 0) && (p.x_sd % VEC == 0) &&
                            (p.out_sb % VEC == 0) && (p.out_sd % VEC == 0) && (p.seqlen >= VEC);
        if (vec_ok) {
            const int64_t n = (int64_t)p.batch * p.dim * (p.seqlen / VEC);
            conv_fwd_seqc_kernel<T, VEC><<<(unsigned)((n + 127) / 128), 128, 0, s>>>(p);
        } else {
            const int64_t n = (int64_t)p.batch * p.dim * p.seqlen;
            conv_fwd_seqc_kernel<T, 1><<<(unsigned)((n + 127) / 128), 128, 0, s>>>(p);
        }
    } else {
        // token-major: a thread owns DV adjacent channels.  4 channels (8-byte vectors for 16-bit types) keep the
        // kernel at ~70 registers -> 6+ CTAs/SM; 8 channels needed 128-182 registers (ncu round 1: 12 % occupancy,
        // 202 us for 335 MB).
        static int dv_env = -1;        // tuning knob: channels per thread (ZG_CONV_VEC = 2 | 4 | 8)
        if (dv_env < 0) { const char *e = getenv("ZG_CONV_VEC"); dv_env = e ? atoi(e) : 0; }
        if (dv_env == 2 || (dv_env == 8 && sizeof(T) == 2)) {
            const int dv = dv_env;
            const bool ok = (p.dim % dv == 0) && (align_bits % (dv * sizeof(T)) == 0) && (p.x_sb % dv == 0) && (p.x_sl % dv == 0) &&
                            (p.out_sb % dv == 0) && (p.out_sl % dv == 0);
            if (ok) {
                const int nchunk2 = (p.seqlen + CONV_LCH - 1) / CONV_LCH;
                const int64_t n = (int64_t)p.batch * nchunk2 * (p.dim / dv);
                if (dv == 2) conv_fwd_dimc_kernel<T, 2><<<(unsigned)((n + 127) / 128), 128, 0, s>>>(p);
                else conv_fwd_dimc_kernel<T, (sizeof(T) == 2 ? 8 : 4)><<<(unsigned)((n + 127) / 128), 128, 0, s>>>(p);
                zg_count_launch();
                return zg_check_launch("causal_conv1d_fwd");
            }
        }
        if constexpr (sizeof(T) == 2) {
            const bool fast = (dv_env == 0 || p.seg_len > 0) && (p.seg_len % CONV_RB == 0) && (p.seg_len == 0 || p.seqlen % p.seg_len == 0) && (p.dim % 4 == 0) && (align_bits % 8 == 0) && (p.x_sb % 4 == 0) && (p.x_sl % 4 == 0) &&
                              (p.out_sb % 4 == 0) && (p.out_sl % 4 == 0) && (p.seqlen % CONV_LCH == 0) &&
                              ((int64_t)p.seqlen * p.x_sl < 0x7fffffffLL) && ((int64_t)p.seqlen * p.out_sl < 0x7fffffffLL);
            // ZG_CONV_SMEM=1: the cp.async-staged kernel (8 channels per lane) where the shape allows; ZG_CONV_SMEM_LCH = 16 | 32 | 64 tokens
            // per warp (read per call, like ZG_SCAN_WP, so that a test can compare both kernels in one process)
            const char *smem_e = getenv("ZG_CONV_SMEM"), *smem_l = getenv("ZG_CONV_SMEM_LCH");
            const int smem_env = smem_e ? atoi(smem_e) : ZG_CONV_SMEM_DEFAULT, smem_lch = smem_l ? atoi(smem_l) : 32;
            if (fast && smem_env == 1 && (smem_lch == 16 || smem_lch == 32 || smem_lch == 64) && (p.dim % CS_CH == 0) && (align_bits % 16 == 0) && (p.x_sb % 8 == 0) &&
                (p.x_sl % 8 == 0) && (p.out_sb % 8 == 0) && (p.out_sl % 8 == 0) && (p.seqlen % smem_lch == 0)) {
                const int64_t nwarp = (int64_t)p.batch * (p.seqlen / smem_lch) * (p.dim / CS_CH);
                const unsigned grid = (unsigned)((nwarp + CS_WARPS - 1) / CS_WARPS);
                constexpr int SMEM = CS_WARPS * CS_WARP_BYTES;      // 48 KB: the default dynamic limit, no attribute needed
                if (smem_lch == 16) conv_fwd_tok8s_kernel<T, 16><<<grid, 32 * CS_WARPS, SMEM, s>>>(p);
                else if (smem_lch == 32) conv_fwd_tok8s_kernel<T, 32><<<grid, 32 * CS_WARPS, SMEM, s>>>(p);
                else conv_fwd_tok8s_kernel<T, 64><<<grid, 32 * CS_WARPS, SMEM, s>>>(p);
                zg_count_launch();
                return zg_check_launch("causal_conv1d_fwd(smem)");
            }
            if (fast) {
                const int64_t n = (int64_t)p.batch * (p.seqlen / CONV_LCH) * (p.dim / 4);
                conv_fwd_tok4_kernel<T><<<(unsigned)((n + 127) / 128), 128, 0, s>>>(p);
                zg_count_launch();
                return zg_check_launch("causal_conv1d_fwd");
            }
        }
        if (p.seg_len > 0)
            return zg_set_error("causal_conv1d_fwd: seg_len needs the 16-bit fast path (seg_len %% 8 == 0 dividing seqlen, seqlen %% 32 == 0, dim %% 4 == 0, 8-byte aligned rows)");
        constexpr int DV = 4;
        constexpr int DB = DV * (int)sizeof(T);
        const bool vec_ok = (p.dim % DV == 0) && (align_bits % DB == 0) && (p.x_sb % DV == 0) && (p.x_sl % DV == 0) &&
                            (p.out_sb % DV == 0) && (p.out_sl % DV == 0);
        const int nchunk = (p.seqlen + CONV_LCH - 1) / CONV_LCH;
        if (vec_ok) {
            const int64_t n = (int64_t)p.batch * nchunk * (p.dim / DV);
            conv_fwd_dimc_kernel<T, DV><<<(unsigned)((n + 127) / 128), 128, 0, s>>>(p);
        } else {
            const int64_t n = (int64_t)p.batch * nchunk * p.dim;
            conv_fwd_dimc_kernel<T, 1><<<(unsigned)((n + 127) / 128), 128, 0, s>>>(p);
        }
    }
    zg_count_launch();
    return zg_check_launch("causal_conv1d_fwd");
}

}  // namespace zg

static int conv_validate(const zg_conv_params &p, const char *who) {
    ZG_REQUIRE(p.dtype == ZG_F32 || p.dtype == ZG_F16 || p.dtype == ZG_BF16, "%s: bad dtype %d", who, p.dtype);
    ZG_REQUIRE(p.wdtype == ZG_F32 || p.wdtype == ZG_F16 || p.wdtype == ZG_BF16, "%s: bad weight dtype %d", who, p.wdtype);
    ZG_REQUIRE(p.width >= 2 && p.width <= 4, "%s only supports width between 2 and 4, got %d", who, p.width);
    ZG_REQUIRE(p.batch >= 0 && p.dim > 0 && p.seqlen >= 0, "%s: bad shape (%d, %d, %d)", who, p.batch, p.dim, p.seqlen);
    ZG_REQUIRE(p.x && p.weight && p.out, "%s: null tensor pointer", who);
    ZG_REQUIRE((p.x_sl == 1 && p.out_sl == 1) || (p.x_sd == 1 && p.out_sd == 1),
               "%s: x and out must both be seq-contiguous or both dim-contiguous", who);
    return 0;
}

extern "C" int zg_causal_conv1d_fwd(const zg_conv_params *pp, void *stream) {
    ZG_REQUIRE(pp != nullptr, "causal_conv1d_fwd: null params");
    const zg_conv_params &p = *pp;
    if (int rc = conv_validate(p, "causal_conv1d_fwd")) return rc;
    const bool seq = (p.x_sl == 1 && p.out_sl == 1);
    ZG_REQUIRE(!(seq && p.x_rowmap), "causal_conv1d_fwd: x_rowmap needs the dim-contiguous layout");
    ZG_REQUIRE(p.seg_len >= 0 && !(seq && p.seg_len > 0), "causal_conv1d_fwd: seg_len needs the dim-contiguous layout");
    if (p.batch == 0 || p.seqlen == 0) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    switch (p.dtype) {
        case ZG_F32: return zg::conv_fwd_t<float>(p, seq, s);
        case ZG_F16: return zg::conv_fwd_t<__half>(p, seq, s);
        default: return zg::conv_fwd_t<__nv_bfloat16>(p, seq, s);
    }
}

// which backward kernel family runs a call (host arithmetic only; the launch and the deterministic workspace query share it)
enum { CONV_BWD_TOK4 = 0, CONV_BWD_TOK = 1, CONV_BWD_SEQC = 2 };
static int conv_bwd_kind(const zg_conv_bwd_params &q) {
    const zg_conv_params &p = q.fwd;
    if (!(p.x_sd == 1 && q.dout_sd == 1 && q.dx_sd == 1 && !(p.x_sl == 1 && p.dim > 1))) return CONV_BWD_SEQC;
    const int esz = zg_dtype_size(p.dtype);
    const uintptr_t al = reinterpret_cast<uintptr_t>(p.x) | reinterpret_cast<uintptr_t>(q.dout) | reinterpret_cast<uintptr_t>(q.dx);
    const int64_t so = p.x_sb | p.x_sl | q.dout_sb | q.dout_sl | q.dx_sb | q.dx_sl;
    const bool vec = (p.dim % 4 == 0) && (al % (4 * esz) == 0) && (so % 4 == 0);
    static int fast4 = -1;             // ZG_CONV_BWD_FAST=0 disables the branch-free 16-bit kernel
    if (fast4 < 0) { const char *e = getenv("ZG_CONV_BWD_FAST"); fast4 = e ? atoi(e) : 1; }
    if (fast4 && esz == 2 && vec && p.seqlen % zg::CONV_B4_LCH == 0 && p.seqlen >= zg::CONV_B4_LCH &&
        (int64_t)p.seqlen * p.x_sl < 0x7fffffffLL && (int64_t)p.seqlen * q.dout_sl < 0x7fffffffLL && (int64_t)p.seqlen * q.dx_sl < 0x7fffffffLL)
        return CONV_BWD_TOK4;
    return CONV_BWD_TOK;
}

static int conv_bwd_validate(const zg_conv_bwd_params &q) {
    if (int rc = conv_validate(q.fwd, "causal_conv1d_bwd")) return rc;
    ZG_REQUIRE(q.dout && q.dx && q.dweight, "causal_conv1d_bwd: null tensor pointer");
    ZG_REQUIRE(q.fwd.seg_len == 0, "causal_conv1d_bwd: seg_len is a forward (sampling) feature");
    return 0;
}

template <bool DET> static int conv_bwd_launch(const zg_conv_bwd_params &q, cudaStream_t s) {
    const zg_conv_params &p = q.fwd;
    const int kind = conv_bwd_kind(q);
    if (kind != CONV_BWD_SEQC) {
        // token-major: DV channels per thread when everything is DV-aligned
        const int esz = zg_dtype_size(p.dtype);
        const uintptr_t al = reinterpret_cast<uintptr_t>(p.x) | reinterpret_cast<uintptr_t>(q.dout) | reinterpret_cast<uintptr_t>(q.dx);
        const int64_t so = p.x_sb | p.x_sl | q.dout_sb | q.dout_sl | q.dx_sb | q.dx_sl;
        const bool vec = (p.dim % 4 == 0) && (al % (4 * esz) == 0) && (so % 4 == 0);
        if (kind == CONV_BWD_TOK4) {
            const int nvb4 = (p.dim / 4 + 31) / 32;
            const int64_t g4 = (int64_t)nvb4 * (((int64_t)p.batch * (p.seqlen / zg::CONV_B4_LCH) + 3) / 4);
            ZG_REQUIRE(g4 <= 0x7fffffffLL, "causal_conv1d_bwd: grid too large");
            if (p.dtype == ZG_BF16) {
                if (p.x_rowmap) zg::conv_bwd_tok4_kernel<__nv_bfloat16, true, DET><<<(unsigned)g4, 128, 0, s>>>(q);
                else zg::conv_bwd_tok4_kernel<__nv_bfloat16, false, DET><<<(unsigned)g4, 128, 0, s>>>(q);
            } else {
                if (p.x_rowmap) zg::conv_bwd_tok4_kernel<__half, true, DET><<<(unsigned)g4, 128, 0, s>>>(q);
                else zg::conv_bwd_tok4_kernel<__half, false, DET><<<(unsigned)g4, 128, 0, s>>>(q);
            }
            zg_count_launch();
            return zg_check_launch("causal_conv1d_bwd(token-major, fast)");
        }
        static int brb = -1, dvs = -1;     // tuning knobs: rows per batch of loads (ZG_CONV_BWD_RB), channels per thread (ZG_CONV_BWD_DV = 2 | 4)
        if (brb < 0) { const char *e = getenv("ZG_CONV_BWD_RB"); brb = e ? atoi(e) : 4; }
        if (dvs < 0) { const char *e = getenv("ZG_CONV_BWD_DV"); dvs = e ? atoi(e) : 2; }
        const int dv = vec ? (dvs == 2 ? 2 : 4) : 1;
        const int nvb = (p.dim / dv + 31) / 32;
        const int nchunk = (p.seqlen + zg::CONV_BLCH - 1) / zg::CONV_BLCH;
        const int64_t grid = (int64_t)nvb * (((int64_t)p.batch * nchunk + 3) / 4);
        ZG_REQUIRE(grid <= 0x7fffffffLL, "causal_conv1d_bwd: grid too large");
#define ZG_CONV_BWD_TOK(TT)                                                                                  \
        do {                                                                                                 \
            if (vec && dvs == 2 && brb == 4) zg::conv_bwd_tok_kernel<TT, 2, 4, DET><<<(unsigned)grid, 128, 0, s>>>(q);      \
            else if (vec && dvs == 2) zg::conv_bwd_tok_kernel<TT, 2, 8, DET><<<(unsigned)grid, 128, 0, s>>>(q);             \
            else if (vec && brb == 2) zg::conv_bwd_tok_kernel<TT, 4, 2, DET><<<(unsigned)grid, 128, 0, s>>>(q);             \
            else if (vec) zg::conv_bwd_tok_kernel<TT, 4, 4, DET><<<(unsigned)grid, 128, 0, s>>>(q);                        \
            else zg::conv_bwd_tok_kernel<TT, 1, 4, DET><<<(unsigned)grid, 128, 0, s>>>(q);                                \
        } while (0)
        switch (p.dtype) {
            case ZG_F32: ZG_CONV_BWD_TOK(float); break;
            case ZG_F16: ZG_CONV_BWD_TOK(__half); break;
            default: ZG_CONV_BWD_TOK(__nv_bfloat16); break;
        }
#undef ZG_CONV_BWD_TOK
        zg_count_launch();
        return zg_check_launch("causal_conv1d_bwd(token-major)");
    }
    ZG_REQUIRE(q.fwd.x_sl == 1 && q.dout_sl == 1 && q.dx_sl == 1, "causal_conv1d_bwd: tensors must be all seq-contiguous or all dim-contiguous");
    ZG_REQUIRE(q.fwd.x_rowmap == nullptr, "causal_conv1d_bwd: x_rowmap needs the dim-contiguous layout");
    const int64_t nthreads = (int64_t)q.fwd.batch * q.fwd.dim * 32;
    const unsigned grid = (unsigned)((nthreads + 127) / 128);
    const int vec = 16 / zg_dtype_size(p.dtype);
    const uintptr_t al2 = reinterpret_cast<uintptr_t>(p.x) | reinterpret_cast<uintptr_t>(q.dout) | reinterpret_cast<uintptr_t>(q.dx);
    const int64_t so2 = p.x_sb | p.x_sd | q.dout_sb | q.dout_sd | q.dx_sb | q.dx_sd;
    const bool fast = (p.seqlen % vec == 0) && (al2 % 16 == 0) && (so2 % vec == 0);
    switch (q.fwd.dtype) {
        case ZG_F32: if (fast) zg::conv_bwd_seqc_vec_kernel<float, DET><<<grid, 128, 0, s>>>(q); else zg::conv_bwd_seqc_kernel<float, DET><<<grid, 128, 0, s>>>(q); break;
        case ZG_F16: if (fast) zg::conv_bwd_seqc_vec_kernel<__half, DET><<<grid, 128, 0, s>>>(q); else zg::conv_bwd_seqc_kernel<__half, DET><<<grid, 128, 0, s>>>(q); break;
        default: if (fast) zg::conv_bwd_seqc_vec_kernel<__nv_bfloat16, DET><<<grid, 128, 0, s>>>(q); else zg::conv_bwd_seqc_kernel<__nv_bfloat16, DET><<<grid, 128, 0, s>>>(q); break;
    }
    zg_count_launch();
    return zg_check_launch("causal_conv1d_bwd");
}

// partial-row regions of the deterministic backward (see the DET notes of the kernels): one row per batch row
// (channel-first) or per 4 consecutive (batch, chunk) rows (token-major: 32-position chunks in the fast kernel, 64 otherwise)
static ZgDetLayout conv_bwd_det_layout(const zg_conv_bwd_params &q, void *ws) {
    const zg_conv_params &p = q.fwd;
    ZgDetLayout lay;
    lay.ws = static_cast<unsigned char *>(ws);
    if (p.batch <= 0 || p.seqlen <= 0 || p.dim <= 0) return lay;
    const int kind = conv_bwd_kind(q);
    const int64_t rows = kind == CONV_BWD_SEQC ? p.batch
                       : ((int64_t)p.batch * (kind == CONV_BWD_TOK4 ? p.seqlen / zg::CONV_B4_LCH : (p.seqlen + zg::CONV_BLCH - 1) / zg::CONV_BLCH) + 3) / 4;
    lay.add(q.dweight, rows, (int64_t)p.dim * p.width);
    lay.add(q.dbias, rows, p.dim);
    return lay;
}

extern "C" int64_t zg_causal_conv1d_bwd_det_workspace_bytes(const zg_conv_bwd_params *q) {
    return q ? conv_bwd_det_layout(*q, nullptr).bytes : 0;
}

extern "C" int zg_causal_conv1d_bwd_det(const zg_conv_bwd_params *qq, void *workspace, int64_t workspace_bytes, void *stream) {
    ZG_REQUIRE(qq != nullptr, "causal_conv1d_bwd_det: null params");
    if (int rc = conv_bwd_validate(*qq)) return rc;
    if (qq->fwd.batch == 0 || qq->fwd.seqlen == 0) return 0;
    const ZgDetLayout lay = conv_bwd_det_layout(*qq, workspace);
    ZG_REQUIRE_WORKSPACE(lay, workspace, workspace_bytes, "causal_conv1d_bwd_det");
    zg_conv_bwd_params q = *qq;                 // the kernel writes partial rows; the reduction adds them to the outputs
    q.dweight = lay.reg[0].part;
    if (q.dbias) q.dbias = lay.reg[1].part;
    cudaStream_t s = (cudaStream_t)stream;
    if (int rc = conv_bwd_launch<true>(q, s)) return rc;
    return lay.reduce(s);
}

extern "C" int zg_causal_conv1d_bwd(const zg_conv_bwd_params *qq, void *stream) {
    ZG_REQUIRE(qq != nullptr, "causal_conv1d_bwd: null params");
    if (int rc = conv_bwd_validate(*qq)) return rc;
    if (qq->fwd.batch == 0 || qq->fwd.seqlen == 0) return 0;
    return conv_bwd_launch<false>(*qq, (cudaStream_t)stream);
}
