// Fused residual-add + RMSNorm/LayerNorm (forward, backward) and the fused ZigMa block tail, sm_90a.
//
// Replaces the Triton kernels _layer_norm_fwd_1pass_kernel / _layer_norm_bwd_kernel
// (dis_mamba/mamba_ssm/ops/triton/layernorm.py:64-120,195-290) and, for the inference fast path,
// the chain of unfused elementwise ops around them in Block.forward (model_zigma.py:416-445).
// HBM-bound: one warp per token row, 16-byte vector loads, the fp32 row lives in registers between
// the statistics pass and the normalisation pass (single global read of every operand).
#include "zg_common.cuh"
#include <stdlib.h>

namespace zg {

// generic element access by runtime dtype (used for (B, D)-sized modulation vectors and weights)
__device__ __forceinline__ float ld_dt(const void *p, int64_t i, int dt) {
    if (dt == ZG_F32) return reinterpret_cast<const float *>(p)[i];
    if (dt == ZG_F16) return __half2float(reinterpret_cast<const __half *>(p)[i]);
    return __bfloat162float(reinterpret_cast<const __nv_bfloat16 *>(p)[i]);
}
__device__ __forceinline__ void st_dt(void *p, int64_t i, int dt, float v) {
    if (dt == ZG_F32) reinterpret_cast<float *>(p)[i] = v;
    else if (dt == ZG_F16) reinterpret_cast<__half *>(p)[i] = __float2half_rn(v);
    else reinterpret_cast<__nv_bfloat16 *>(p)[i] = __float2bfloat16_rn(v);
}
template <typename T> __device__ __forceinline__ float round_to(float v) { return zg_to_float<T>(zg_from_float<T>(v)); }

// 4 consecutive elements starting at i (i % 4 == 0, pointers 16B/8B aligned by contract)
template <typename T> __device__ __forceinline__ void ld4(const T *p, int64_t i, float (&o)[4]);
template <> __device__ __forceinline__ void ld4<float>(const float *p, int64_t i, float (&o)[4]) {
    float4 v = *reinterpret_cast<const float4 *>(p + i);
    o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
}
template <> __device__ __forceinline__ void ld4<__nv_bfloat16>(const __nv_bfloat16 *p, int64_t i, float (&o)[4]) {
    uint2 v = *reinterpret_cast<const uint2 *>(p + i);
    o[0] = __uint_as_float(v.x << 16); o[1] = __uint_as_float(v.x & 0xffff0000u);
    o[2] = __uint_as_float(v.y << 16); o[3] = __uint_as_float(v.y & 0xffff0000u);
}
template <> __device__ __forceinline__ void ld4<__half>(const __half *p, int64_t i, float (&o)[4]) {
    uint2 v = *reinterpret_cast<const uint2 *>(p + i);
    float2 a = __half22float2(*reinterpret_cast<__half2 *>(&v.x)), b = __half22float2(*reinterpret_cast<__half2 *>(&v.y));
    o[0] = a.x; o[1] = a.y; o[2] = b.x; o[3] = b.y;
}
template <typename T> __device__ __forceinline__ void st4(T *p, int64_t i, const float (&o)[4]);
template <> __device__ __forceinline__ void st4<float>(float *p, int64_t i, const float (&o)[4]) {
    *reinterpret_cast<float4 *>(p + i) = make_float4(o[0], o[1], o[2], o[3]);
}
template <> __device__ __forceinline__ void st4<__nv_bfloat16>(__nv_bfloat16 *p, int64_t i, const float (&o)[4]) {
    __nv_bfloat162 a = __floats2bfloat162_rn(o[0], o[1]), b = __floats2bfloat162_rn(o[2], o[3]);
    uint2 v; v.x = *reinterpret_cast<unsigned *>(&a); v.y = *reinterpret_cast<unsigned *>(&b);
    *reinterpret_cast<uint2 *>(p + i) = v;
}
template <> __device__ __forceinline__ void st4<__half>(__half *p, int64_t i, const float (&o)[4]) {
    __half2 a = __floats2half2_rn(o[0], o[1]), b = __floats2half2_rn(o[2], o[3]);
    uint2 v; v.x = *reinterpret_cast<unsigned *>(&a); v.y = *reinterpret_cast<unsigned *>(&b);
    *reinterpret_cast<uint2 *>(p + i) = v;
}

constexpr int NORM_MAXQ = 16;   // quads (4 elements) per lane held in registers -> ncols <= 2048

// ------------------------------------------------------------------------------------------------
// add + norm forward.  T = x/y dtype, R = residual dtype.  Requires ncols % 4 == 0, ncols <= 2048.
template <typename T, typename R>
__global__ void __launch_bounds__(128) add_norm_fwd_kernel(const zg_norm_params p) {
    const int row = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= p.nrows) return;
    const int N = p.ncols, nq = N >> 2;
    const T *x = reinterpret_cast<const T *>(p.x) + (int64_t)row * p.x_rs;
    const R *res = p.residual ? reinterpret_cast<const R *>(p.residual) + (int64_t)row * p.res_rs : nullptr;
    R *rout = p.residual_out ? reinterpret_cast<R *>(p.residual_out) + (int64_t)row * p.resout_rs : nullptr;
    T *y = reinterpret_cast<T *>(p.y) + (int64_t)row * p.y_rs;
    float r[NORM_MAXQ][4];
    float sum = 0.f, sumsq = 0.f;
#pragma unroll
    for (int k = 0; k < NORM_MAXQ; ++k) {
        const int q = lane + 32 * k;
        if (q < nq) {
            ld4<T>(x, 4 * q, r[k]);
            if (res) {
                float t[4];
                ld4<R>(res, 4 * q, t);
#pragma unroll
                for (int i = 0; i < 4; ++i) r[k][i] += t[i];
            }
            if (rout) {
                st4<R>(rout, 4 * q, r[k]);
                // the reference stores residual_out in R and normalises the fp32 value (layernorm.py:96-101)
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) { sum += r[k][i]; sumsq += r[k][i] * r[k][i]; }
        }
    }
    float mean = 0.f, var;
    if (p.is_rms) {
        var = zg_warp_sum(sumsq) / N;
    } else {
        mean = zg_warp_sum(sum) / N;
        float s2 = 0.f;
#pragma unroll
        for (int k = 0; k < NORM_MAXQ; ++k)
            if (lane + 32 * k < nq)
#pragma unroll
                for (int i = 0; i < 4; ++i) { const float d = r[k][i] - mean; s2 += d * d; }
        var = zg_warp_sum(s2) / N;
    }
    const float rstd = 1.f / sqrtf(var + p.eps);
    if (lane == 0) {
        if (p.rstd) p.rstd[row] = rstd;
        if (p.mean && !p.is_rms) p.mean[row] = mean;
    }
#pragma unroll
    for (int k = 0; k < NORM_MAXQ; ++k) {
        const int q = lane + 32 * k;
        if (q < nq) {
            float o[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                float v = (r[k][i] - mean) * rstd;
                if (p.weight) v *= ld_dt(p.weight, 4 * q + i, p.wdtype);
                if (p.bias) v += ld_dt(p.bias, 4 * q + i, p.wdtype);
                o[i] = v;
            }
            st4<T>(y, 4 * q, o);
        }
    }
}

// add + norm backward (layernorm.py:195-290).  x = saved residual_out (dtype R), one warp per row;
// dw/db accumulated per CTA in shared memory then atomically into the fp32 outputs.
//   xhat = (x - mean) * rstd;  wdy = dy * w;  c1 = mean(xhat * wdy);  c2 = mean(wdy) (0 for RMS)
//   dx = (wdy - (xhat * c1 + c2)) * rstd (+ dresidual)
// DET: dweight / dbias of p address partial rows, one per warp of the grid -- (gridDim.x * 4, ncols) -- stored, not added
// (zg_add_norm_bwd_det).
template <typename T, typename R, bool DET>
__global__ void __launch_bounds__(128) add_norm_bwd_kernel(const zg_norm_bwd_params p) {
    // persistent warps: each warp walks rows with a grid stride and keeps its dweight/dbias partial
    // sums in registers (lane owns columns lane, lane+32, ...), one atomicAdd per column at the end.
    constexpr int MAXC = 4 * NORM_MAXQ;   // columns per lane
    const int warp = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int nwarps = (int)(((int64_t)gridDim.x * blockDim.x) >> 5);
    const int lane = threadIdx.x & 31;
    const int N = p.ncols;
    float dw[MAXC], db[MAXC];
#pragma unroll
    for (int k = 0; k < MAXC; ++k) { dw[k] = 0.f; db[k] = 0.f; }
    for (int row = warp; row < p.nrows; row += nwarps) {
        const T *dy = reinterpret_cast<const T *>(p.dy) + (int64_t)row * p.dy_rs;
        const R *x = reinterpret_cast<const R *>(p.x) + (int64_t)row * p.x_rs;
        const R *dres = p.dresidual ? reinterpret_cast<const R *>(p.dresidual) + (int64_t)row * p.dres_rs : nullptr;
        T *dx = reinterpret_cast<T *>(p.dx) + (int64_t)row * p.dx_rs;
        R *dresin = p.dresidual_in ? reinterpret_cast<R *>(p.dresidual_in) + (int64_t)row * p.dresin_rs : nullptr;
        const float rstd = p.rstd[row];
        const float mean = (p.is_rms || !p.mean) ? 0.f : p.mean[row];
        float c1 = 0.f, c2 = 0.f;
#pragma unroll
        for (int k = 0; k < MAXC; ++k) {
            const int i = lane + 32 * k;
            if (i < N) {
                const float xhat = (zg_to_float<R>(x[i]) - mean) * rstd;
                const float g = zg_to_float<T>(dy[i]);
                const float wdy = g * (p.weight ? ld_dt(p.weight, i, p.wdtype) : 1.f);
                c1 += xhat * wdy;
                c2 += wdy;
                dw[k] += g * xhat;
                db[k] += g;
            }
        }
        c1 = zg_warp_sum(c1) / N;
        c2 = p.is_rms ? 0.f : zg_warp_sum(c2) / N;
        for (int i = lane; i < N; i += 32) {
            const float xhat = (zg_to_float<R>(x[i]) - mean) * rstd;
            const float wdy = zg_to_float<T>(dy[i]) * (p.weight ? ld_dt(p.weight, i, p.wdtype) : 1.f);
            float d = (wdy - (xhat * c1 + c2)) * rstd;
            if (dres) d += zg_to_float<R>(dres[i]);
            if (dresin) dresin[i] = zg_from_float<R>(d);
            dx[i] = zg_from_float<T>(d);
        }
    }
#pragma unroll
    for (int k = 0; k < MAXC; ++k) {
        const int i = lane + 32 * k;
        if (DET && i < N) {
            if (p.dweight) p.dweight[(int64_t)warp * N + i] = dw[k];
            if (p.dbias) p.dbias[(int64_t)warp * N + i] = db[k];
        } else if (i < N) {
            if (p.dweight) atomicAdd(p.dweight + i, dw[k]);
            if (p.dbias) atomicAdd(p.dbias + i, db[k]);
        }
    }
}

// Vectorised backward: MAXQ quads (4 columns) per lane, every row operand fetched ONCE as 8/16-byte vectors
// that stay in registers between the statistics pass and the dx pass; weights preloaded; persistent warps
// with a grid stride keep their dweight/dbias partial sums in registers, summed over the CTA's 4 warps in
// shared memory before the atomics.  (The scalar kernel below remains for unaligned / odd shapes: ncu
// round 1 had it at 0.36 ms for 16384 x 640 -- 2-byte loads, 128 accumulator registers, two dependent
// passes over global memory -- against 0.03 ms of HBM time.)
// DET: dweight / dbias of p address partial rows, one per CTA -- (gridDim.x, ncols) -- stored, not added.
template <typename T, typename R, int MAXQ, bool DET>
__global__ void __launch_bounds__(128) add_norm_bwd_vec_kernel(const zg_norm_bwd_params p) {
    const int warp = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int nwarps = (int)(((int64_t)gridDim.x * blockDim.x) >> 5);
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int N = p.ncols, nq = N >> 2;
    const bool has_db = p.dbias != nullptr;
    float w[MAXQ][4], dw[MAXQ][4], db[MAXQ][4];
#pragma unroll
    for (int k = 0; k < MAXQ; ++k)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int c = 4 * (lane + 32 * k) + i;
            w[k][i] = (p.weight && c < N) ? ld_dt(p.weight, c, p.wdtype) : 1.f;
            dw[k][i] = 0.f; db[k][i] = 0.f;
        }
    const float invN = 1.f / N;
    for (int row = warp; row < p.nrows; row += nwarps) {
        const T *dy = reinterpret_cast<const T *>(p.dy) + (int64_t)row * p.dy_rs;
        const R *x = reinterpret_cast<const R *>(p.x) + (int64_t)row * p.x_rs;
        const R *dres = p.dresidual ? reinterpret_cast<const R *>(p.dresidual) + (int64_t)row * p.dres_rs : nullptr;
        T *dx = reinterpret_cast<T *>(p.dx) + (int64_t)row * p.dx_rs;
        R *dresin = p.dresidual_in ? reinterpret_cast<R *>(p.dresidual_in) + (int64_t)row * p.dresin_rs : nullptr;
        const float rstd = p.rstd[row];
        const float mean = (p.is_rms || !p.mean) ? 0.f : p.mean[row];
        float xh[MAXQ][4], g[MAXQ][4], dr[MAXQ][4];
#pragma unroll
        for (int k = 0; k < MAXQ; ++k) {
            const int q = lane + 32 * k;
            if (q < nq) {
                ld4<R>(x, 4 * q, xh[k]);
                ld4<T>(dy, 4 * q, g[k]);
                if (dres) ld4<R>(dres, 4 * q, dr[k]);
            }
        }
        float c1 = 0.f, c2 = 0.f;
#pragma unroll
        for (int k = 0; k < MAXQ; ++k) {
            if (lane + 32 * k < nq) {
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    xh[k][i] = (xh[k][i] - mean) * rstd;
                    const float wdy = g[k][i] * w[k][i];
                    c1 = fmaf(xh[k][i], wdy, c1);
                    c2 += wdy;
                    dw[k][i] = fmaf(g[k][i], xh[k][i], dw[k][i]);
                    if (has_db) db[k][i] += g[k][i];
                }
            }
        }
        c1 = zg_warp_sum(c1) * invN;
        c2 = p.is_rms ? 0.f : zg_warp_sum(c2) * invN;
#pragma unroll
        for (int k = 0; k < MAXQ; ++k) {
            const int q = lane + 32 * k;
            if (q < nq) {
                float o[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    float d = (g[k][i] * w[k][i] - (xh[k][i] * c1 + c2)) * rstd;
                    if (dres) d += dr[k][i];
                    o[i] = d;
                }
                if (dresin) st4<R>(dresin, 4 * q, o);
                st4<T>(dx, 4 * q, o);
            }
        }
    }
    // CTA reduction (4 warps) then one atomic per column per CTA
    __shared__ float red[4][128 * MAXQ];
    for (int pass = 0; pass < 2; ++pass) {
        if (pass == 1 && !has_db) break;
        if (pass == 0 && !p.dweight) continue;
        __syncthreads();
#pragma unroll
        for (int k = 0; k < MAXQ; ++k)
#pragma unroll
            for (int i = 0; i < 4; ++i) red[wib][4 * (lane + 32 * k) + i] = pass ? db[k][i] : dw[k][i];
        __syncthreads();
        float *dst = pass ? p.dbias : p.dweight;
        if constexpr (DET) {
            for (int c = threadIdx.x; c < N; c += 128) dst[(int64_t)blockIdx.x * N + c] = red[0][c] + red[1][c] + red[2][c] + red[3][c];
        } else {
            for (int c = threadIdx.x; c < N; c += 128) atomicAdd(dst + c, red[0][c] + red[1][c] + red[2][c] + red[3][c]);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Block tail (see include/zigma_b200.h).  One warp per token; all row operands are read exactly once.
// MAXQ = quads (4 elements) per lane: D <= 128 * MAXQ.  The row operands are first pulled into registers
// as RAW 8/16-byte vectors (all loads of a row in flight together -- the kernel is pure HBM streaming,
// ~670 MB per call at BASELINE config 2), only then converted and combined.
template <typename T> struct Raw4 { uint2 v; };                 // 4 x 16-bit
template <> struct Raw4<float> { float4 v; };
template <typename T> __device__ __forceinline__ Raw4<T> ldraw(const T *p, int64_t i) {
    Raw4<T> r;
    r.v = *reinterpret_cast<const decltype(r.v) *>(p + i);
    return r;
}
template <typename T> __device__ __forceinline__ Raw4<T> raw_ones();       // four 1.0 in the storage format
template <> __device__ __forceinline__ Raw4<float> raw_ones<float>() { Raw4<float> r; r.v = make_float4(1.f, 1.f, 1.f, 1.f); return r; }
template <> __device__ __forceinline__ Raw4<__nv_bfloat16> raw_ones<__nv_bfloat16>() { Raw4<__nv_bfloat16> r; r.v = make_uint2(0x3f803f80u, 0x3f803f80u); return r; }
template <> __device__ __forceinline__ Raw4<__half> raw_ones<__half>() { Raw4<__half> r; r.v = make_uint2(0x3c003c00u, 0x3c003c00u); return r; }
template <typename T> __device__ __forceinline__ void cvt4(const Raw4<T> &r, float (&o)[4]);
template <> __device__ __forceinline__ void cvt4<float>(const Raw4<float> &r, float (&o)[4]) {
    o[0] = r.v.x; o[1] = r.v.y; o[2] = r.v.z; o[3] = r.v.w;
}
template <> __device__ __forceinline__ void cvt4<__nv_bfloat16>(const Raw4<__nv_bfloat16> &r, float (&o)[4]) {
    o[0] = __uint_as_float(r.v.x << 16); o[1] = __uint_as_float(r.v.x & 0xffff0000u);
    o[2] = __uint_as_float(r.v.y << 16); o[3] = __uint_as_float(r.v.y & 0xffff0000u);
}
template <> __device__ __forceinline__ void cvt4<__half>(const Raw4<__half> &r, float (&o)[4]) {
    uint2 v = r.v;
    float2 a = __half22float2(*reinterpret_cast<__half2 *>(&v.x)), b = __half22float2(*reinterpret_cast<__half2 *>(&v.y));
    o[0] = a.x; o[1] = a.y; o[2] = b.x; o[3] = b.y;
}

template <typename T, int MAXQ>
__global__ void __launch_bounds__(128, (MAXQ <= 6) ? 6 : 1) block_tail_kernel(const zg_block_tail_params p) {
    const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    const int64_t nrows = (int64_t)p.batch * p.seqlen;
    if (row >= nrows) return;
    const int D = p.dim, nq = D >> 2;
    const int b = (int)(row / p.seqlen), l = (int)(row % p.seqlen);
    const T *x = reinterpret_cast<const T *>(p.x) + row * D;
    const T *mix = nullptr;
    if (p.mix) {
        const int64_t src = (int64_t)b * p.seqlen + (p.rowmap ? p.rowmap[l] : l);
        mix = reinterpret_cast<const T *>(p.mix) + src * D;
    }
    const T *gate = p.gate ? reinterpret_cast<const T *>(p.gate) + (int64_t)b * p.mod_rs : nullptr;
    const T *shift = p.shift ? reinterpret_cast<const T *>(p.shift) + (int64_t)b * p.mod_rs : nullptr;
    const T *scale = p.scale ? reinterpret_cast<const T *>(p.scale) + (int64_t)b * p.mod_rs : nullptr;
    const T *nw = reinterpret_cast<const T *>(p.norm_w);
    const float *res = p.residual ? p.residual + row * D : nullptr;
    float *rout = p.residual_out ? p.residual_out + row * D : nullptr;
    T *normed = reinterpret_cast<T *>(p.normed) + row * D;
    T *modded = p.modded ? reinterpret_cast<T *>(p.modded) + row * D : nullptr;

    // ---- phase 1: every streaming load of the row, back to back ---------------------------------------
    Raw4<T> rx[MAXQ], rm[MAXQ];
    float4 rr[MAXQ];
#pragma unroll
    for (int k = 0; k < MAXQ; ++k) {
        const int q = lane + 32 * k;
        if (q < nq) {
            rx[k] = ldraw<T>(x, 4 * q);
            if (mix) rm[k] = ldraw<T>(mix, 4 * q);
            if (res) rr[k] = *reinterpret_cast<const float4 *>(res + 4 * q);
        }
    }
    // ---- phase 2: hidden = x + gate * mix; r = residual + hidden; statistics -------------------------
    float r[MAXQ][4];
    float sumsq = 0.f;
#pragma unroll
    for (int k = 0; k < MAXQ; ++k) {
        const int q = lane + 32 * k;
        if (q < nq) {
            cvt4<T>(rx[k], r[k]);
            if (mix) {
                float m[4], g[4];
                cvt4<T>(rm[k], m);
                ld4<T>(gate, 4 * q, g);
#pragma unroll
                for (int i = 0; i < 4; ++i)   // x + gate * mixer(...)  each op rounded to T as in eager torch
                    r[k][i] = round_to<T>(r[k][i] + round_to<T>(g[i] * m[i]));
            }
            if (res) {
                r[k][0] += rr[k].x; r[k][1] += rr[k].y; r[k][2] += rr[k].z; r[k][3] += rr[k].w;
            }
            if (rout) st4<float>(rout, 4 * q, r[k]);
#pragma unroll
            for (int i = 0; i < 4; ++i) sumsq += r[k][i] * r[k][i];
        }
    }
    const float rstd = 1.f / sqrtf(zg_warp_sum(sumsq) / D + p.eps);
    if (p.rstd && lane == 0) p.rstd[row] = rstd;
    float sum2 = 0.f;
#pragma unroll
    for (int k = 0; k < MAXQ; ++k) {
        const int q = lane + 32 * k;
        if (q < nq) {
            float w[4];
            ld4<T>(nw, 4 * q, w);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                r[k][i] = round_to<T>(r[k][i] * rstd * w[i]);   // RMSNorm output as stored by the reference
                sum2 += r[k][i];
            }
        }
    }
    if (p.final_layer) {
        // norm_final = LayerNorm(no affine, eps 1e-6) on the materialised norm_f output (model_zigma.py:320,335)
        const float mean = zg_warp_sum(sum2) / D;
        float s2 = 0.f;
#pragma unroll
        for (int k = 0; k < MAXQ; ++k)
            if (lane + 32 * k < nq)
#pragma unroll
                for (int i = 0; i < 4; ++i) { const float d = r[k][i] - mean; s2 += d * d; }
        const float rstd2 = 1.f / sqrtf(zg_warp_sum(s2) / D + 1e-6f);
#pragma unroll
        for (int k = 0; k < MAXQ; ++k) {
            const int q = lane + 32 * k;
            if (q < nq) {
                float o[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) o[i] = (r[k][i] - mean) * rstd2;
                st4<T>(normed, 4 * q, o);
            }
        }
        return;
    }
#pragma unroll
    for (int k = 0; k < MAXQ; ++k) {
        const int q = lane + 32 * k;
        if (q < nq) {
            st4<T>(normed, 4 * q, r[k]);
            if (modded) {
                float sc[4], sh[4], o[4];
                ld4<T>(scale, 4 * q, sc);
                ld4<T>(shift, 4 * q, sh);
#pragma unroll
                for (int i = 0; i < 4; ++i)   // x * (1 + scale) + shift, eager-torch rounding points
                    o[i] = round_to<T>(r[k][i] * round_to<T>(1.f + sc[i])) + sh[i];
                st4<T>(modded, 4 * q, o);
            }
        }
    }
}

#ifndef ZG_TAIL_PREFETCH_MOD
#define ZG_TAIL_PREFETCH_MOD 1
#endif
#ifndef ZG_TAIL_MINB
#define ZG_TAIL_MINB 12
#endif
// Round 2: FOUR warps per row (one 128-thread CTA = one token row).  The one-warp-per-row kernel above keeps a whole row in the
// registers of 32 lanes (67 registers at D = 640 -> 7 CTAs = 28 warps per SM, 42 % occupancy) and ncu shows it purely
// latency-bound: long_scoreboard 12.9 warps per issue, issue 36 %.  Spreading the row
// over 128 lanes leaves 1-2 quads per lane (about half the registers, twice the resident warps) at the price of one
// shared-memory reduction per statistic.  Same arithmetic and rounding points.  Measured at config 2 (672 MB per call):
// 149.7 us (one warp per row) -> 136.5 us (this kernel, 40 registers, 12 CTAs / SM) -> 121.1 us = 5.54 TB/s = 0.84 of the measured
// HBM peak with the scale / shift rows prefetched too (ZG_TAIL_PREFETCH_MOD); 32 registers / 16 CTAs without that prefetch: 122.0 us.
// PE (zg_block_tail_fwd_pe, the first tail of a forward): mix is the (seqlen, dim) positional-embedding table shared by every
// batch element and there is no gate: hidden = round(tokens + pos_embed), the reference's `x = x + self.pos_embed`
// (model_zigma.py:941), without an elementwise pass of its own.  A separate instantiation: the per-layer instance is unchanged.
// DP (zg_block_tail_fwd_dp, stochastic depth in training): hidden is multiplied by the batch element's drop-path multiplier
// before the residual add, kept = round(hidden * path_scale[b]), the reference's eager `x * mask`.  One scalar load per row.
// RB (zg_block_tail_fwd_rebuild): x is not read; it is the previous tail's normed output, rebuilt from the residual row this
// kernel loads anyway as round(residual * x_rstd[row] * x_norm_w), the previous tail's own expression on the same operands.
template <typename T, int MAXQ, bool PE, bool DP, bool RB = false>
__device__ __forceinline__ void block_tail_row4_body(const zg_block_tail_params &p, const void *path_scale, const float *x_rstd = nullptr,
                                                     const void *x_norm_w = nullptr) {
    __shared__ float red[3][4];
    const int64_t row = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int D = p.dim, nq = D >> 2;
    const int b = (int)(row / p.seqlen), l = (int)(row % p.seqlen);
    const T *x = RB ? reinterpret_cast<const T *>(x_norm_w) : reinterpret_cast<const T *>(p.x) + row * D;   // RB: per column
    const T *mix = nullptr;
    if (p.mix) {
        const int64_t src = (PE ? 0 : (int64_t)b * p.seqlen) + (p.rowmap ? p.rowmap[l] : l);
        mix = reinterpret_cast<const T *>(p.mix) + src * D;
    }
    const T *gate = (!PE && p.gate) ? reinterpret_cast<const T *>(p.gate) + (int64_t)b * p.mod_rs : nullptr;
    const T *shift = p.shift ? reinterpret_cast<const T *>(p.shift) + (int64_t)b * p.mod_rs : nullptr;
    const T *scale = p.scale ? reinterpret_cast<const T *>(p.scale) + (int64_t)b * p.mod_rs : nullptr;
    const T *nw = reinterpret_cast<const T *>(p.norm_w);
    const float *res = p.residual ? p.residual + row * D : nullptr;
    float *rout = p.residual_out ? p.residual_out + row * D : nullptr;
    T *normed = reinterpret_cast<T *>(p.normed) + row * D;
    T *modded = p.modded ? reinterpret_cast<T *>(p.modded) + row * D : nullptr;
    auto block_sum = [&](float v, int slot) {
        v = zg_warp_sum(v);
        if (lane == 0) red[slot][warp] = v;
        __syncthreads();
        return (red[slot][0] + red[slot][1]) + (red[slot][2] + red[slot][3]);
    };

    // every load of the row (and of the per-column operands) is issued before the first use
    Raw4<T> rx[MAXQ], rm[MAXQ], rg[MAXQ], rw[MAXQ];
#if ZG_TAIL_PREFETCH_MOD
    Raw4<T> rsc[MAXQ], rsh[MAXQ];
#endif
    float4 rr[MAXQ];
#pragma unroll
    for (int k = 0; k < MAXQ; ++k) {
        const int q = tid + 128 * k;
        if (q < nq) {
            rx[k] = ldraw<T>(x, 4 * q);
            if (mix) { rm[k] = ldraw<T>(mix, 4 * q); rg[k] = PE ? raw_ones<T>() : ldraw<T>(gate, 4 * q); }     // PE: gate = 1, round(1 * m) = m
            if (RB || res) rr[k] = *reinterpret_cast<const float4 *>(res + 4 * q);
            rw[k] = ldraw<T>(nw, 4 * q);
#if ZG_TAIL_PREFETCH_MOD
            if (!RB && modded) { rsc[k] = ldraw<T>(scale, 4 * q); rsh[k] = ldraw<T>(shift, 4 * q); }   // (RB: 40 registers without spills)
#endif
        }
    }
    float dps = 1.f;
    if constexpr (DP) dps = zg_to_float<T>(reinterpret_cast<const T *>(path_scale)[b]);
    float xrs = 0.f;
    if constexpr (RB) xrs = x_rstd[row];
    float r[MAXQ][4];
    float sumsq = 0.f;
#pragma unroll
    for (int k = 0; k < MAXQ; ++k) {
        const int q = tid + 128 * k;
        if (q < nq) {
            if constexpr (RB) {
                float w[4];
                const float rp[4] = {rr[k].x, rr[k].y, rr[k].z, rr[k].w};
                cvt4<T>(rx[k], w);
#pragma unroll
                for (int i = 0; i < 4; ++i) r[k][i] = round_to<T>(__fmul_rn(__fmul_rn(rp[i], xrs), w[i]));   // no FMA: the stored product
            } else {
                cvt4<T>(rx[k], r[k]);
            }
            if (mix) {
                float m[4], g[4];
                cvt4<T>(rm[k], m);
                cvt4<T>(rg[k], g);
#pragma unroll
                for (int i = 0; i < 4; ++i)   // x + gate * mixer(...)  each op rounded to T as in eager torch
                    r[k][i] = round_to<T>(r[k][i] + round_to<T>(g[i] * m[i]));
            }
            if constexpr (DP) {
#pragma unroll
                for (int i = 0; i < 4; ++i) r[k][i] = round_to<T>(__fmul_rn(r[k][i], dps));   // rounded before the add (no FMA)
            }
            if (RB || res) {
                r[k][0] += rr[k].x; r[k][1] += rr[k].y; r[k][2] += rr[k].z; r[k][3] += rr[k].w;
            }
            if (rout) st4<float>(rout, 4 * q, r[k]);
#pragma unroll
            for (int i = 0; i < 4; ++i) sumsq += r[k][i] * r[k][i];
        }
    }
    const float rstd = 1.f / sqrtf(block_sum(sumsq, 0) / D + p.eps);
    if (p.rstd && tid == 0) p.rstd[row] = rstd;
    float sum2 = 0.f;
#pragma unroll
    for (int k = 0; k < MAXQ; ++k) {
        const int q = tid + 128 * k;
        if (q < nq) {
            float w[4];
            cvt4<T>(rw[k], w);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                r[k][i] = round_to<T>(r[k][i] * rstd * w[i]);   // RMSNorm output as stored by the reference
                sum2 += r[k][i];
            }
        }
    }
    if (!DP && p.final_layer) {      // (the drop-path entry point rejects final_layer)
        // norm_final = LayerNorm(no affine, eps 1e-6) on the materialised norm_f output (model_zigma.py:320,335)
        const float mean = block_sum(sum2, 1) / D;
        float s2 = 0.f;
#pragma unroll
        for (int k = 0; k < MAXQ; ++k)
            if (tid + 128 * k < nq)
#pragma unroll
                for (int i = 0; i < 4; ++i) { const float d = r[k][i] - mean; s2 += d * d; }
        const float rstd2 = 1.f / sqrtf(block_sum(s2, 2) / D + 1e-6f);
#pragma unroll
        for (int k = 0; k < MAXQ; ++k) {
            const int q = tid + 128 * k;
            if (q < nq) {
                float o[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) o[i] = (r[k][i] - mean) * rstd2;
                st4<T>(normed, 4 * q, o);
            }
        }
        return;
    }
#pragma unroll
    for (int k = 0; k < MAXQ; ++k) {
        const int q = tid + 128 * k;
        if (q < nq) {
            if (!RB || p.normed) st4<T>(normed, 4 * q, r[k]);      // (RB: normed may be NULL below the final layer)
            if (modded) {
                float sc[4], sh[4], o[4];
#if ZG_TAIL_PREFETCH_MOD
                if constexpr (RB) {
                    ld4<T>(scale, 4 * q, sc);
                    ld4<T>(shift, 4 * q, sh);
                } else {
                    cvt4<T>(rsc[k], sc);
                    cvt4<T>(rsh[k], sh);
                }
#else
                ld4<T>(scale, 4 * q, sc);
                ld4<T>(shift, 4 * q, sh);
#endif
#pragma unroll
                for (int i = 0; i < 4; ++i)   // x * (1 + scale) + shift, eager-torch rounding points
                    o[i] = round_to<T>(r[k][i] * round_to<T>(1.f + sc[i])) + sh[i];
                st4<T>(modded, 4 * q, o);
            }
        }
    }
}

template <typename T, int MAXQ, bool PE>
__global__ void __launch_bounds__(128, ZG_TAIL_MINB) block_tail_row4_kernel(const zg_block_tail_params p) {
    block_tail_row4_body<T, MAXQ, PE, false>(p, nullptr);
}

template <typename T, int MAXQ>
__global__ void __launch_bounds__(128, ZG_TAIL_MINB) block_tail_dp_fwd_kernel(const zg_block_tail_dp_params p) {
    block_tail_row4_body<T, MAXQ, false, true>(p.base, p.path_scale);
}

template <typename T, int MAXQ>
__global__ void __launch_bounds__(128, ZG_TAIL_MINB) block_tail_rebuild_fwd_kernel(const zg_block_tail_rebuild_params p) {
    block_tail_row4_body<T, MAXQ, false, false, true>(p.base, nullptr, p.x_rstd, p.x_norm_w);
}

// zg_block_tail_fwd_rebuild: the four-warps-per-row kernel only (dim <= 1024 -> Q 1 or 2, checked by the entry point)
template <typename T> static int block_tail_rebuild_t(const zg_block_tail_rebuild_params &p, cudaStream_t s) {
    const unsigned g4 = (unsigned)((int64_t)p.base.batch * p.base.seqlen);
    if (p.base.dim <= 512) block_tail_rebuild_fwd_kernel<T, 1><<<g4, 128, 0, s>>>(p);
    else block_tail_rebuild_fwd_kernel<T, 2><<<g4, 128, 0, s>>>(p);
    zg_count_launch();
    return zg_check_launch("block_tail_fwd_rebuild");
}

// zg_block_tail_fwd_dp: the four-warps-per-row kernel only (dim <= 1024 -> Q 1 or 2, checked by the entry point)
template <typename T> static int block_tail_dp_t(const zg_block_tail_dp_params &p, cudaStream_t s) {
    const unsigned g4 = (unsigned)((int64_t)p.base.batch * p.base.seqlen);
    if (p.base.dim <= 512) block_tail_dp_fwd_kernel<T, 1><<<g4, 128, 0, s>>>(p);
    else block_tail_dp_fwd_kernel<T, 2><<<g4, 128, 0, s>>>(p);
    zg_count_launch();
    return zg_check_launch("block_tail_fwd_dp");
}

template <typename T> static int block_tail_t(const zg_block_tail_params &p, cudaStream_t s, bool pe = false) {
    const int64_t nrows = (int64_t)p.batch * p.seqlen;
    static int row4 = -1;       // ZG_TAIL_ROW4=0: the round-1 kernel (one warp per row)
    if (row4 < 0) { const char *e = getenv("ZG_TAIL_ROW4"); row4 = e ? atoi(e) : 1; }
    if ((row4 || pe) && nrows <= 0x7fffffffLL && p.dim <= 2048) {
        const unsigned g4 = (unsigned)nrows;
#define ZG_TAIL4(Q) do { if (pe) block_tail_row4_kernel<T, Q, true><<<g4, 128, 0, s>>>(p); else block_tail_row4_kernel<T, Q, false><<<g4, 128, 0, s>>>(p); } while (0)
        if (p.dim <= 512) ZG_TAIL4(1);
        else if (p.dim <= 1024) ZG_TAIL4(2);
        else if (p.dim <= 1536) ZG_TAIL4(3);
        else ZG_TAIL4(4);
#undef ZG_TAIL4
        zg_count_launch();
        return zg_check_launch("block_tail_fwd");
    }
    if (pe) return zg_set_error("block_tail_fwd_pe: dim <= 2048 and fewer than 2^31 rows only, got dim %d", p.dim);
    const unsigned grid = (unsigned)((nrows * 32 + 127) / 128);
    // MAXQ = ceil(D / 128) exactly for the model widths of the reference zoo (368, 640, 768, 1024, 1536): the raw
    // operand vectors of a row live in registers, so an over-sized MAXQ costs occupancy (ncu round 1: 92 registers at
    // MAXQ = 8 for D = 640 -> 5 CTAs/SM, 49 % of the HBM roofline)
    if (p.dim <= 512) block_tail_kernel<T, 4><<<grid, 128, 0, s>>>(p);
    else if (p.dim <= 640) block_tail_kernel<T, 5><<<grid, 128, 0, s>>>(p);
    else if (p.dim <= 768) block_tail_kernel<T, 6><<<grid, 128, 0, s>>>(p);
    else if (p.dim <= 1024) block_tail_kernel<T, 8><<<grid, 128, 0, s>>>(p);
    else if (p.dim <= 1536) block_tail_kernel<T, 12><<<grid, 128, 0, s>>>(p);
    else block_tail_kernel<T, NORM_MAXQ><<<grid, 128, 0, s>>>(p);
    zg_count_launch();
    return zg_check_launch("block_tail_fwd");
}

// ------------------------------------------------------------------------------------------------
// Block tail backward (see include/zigma_b200.h).  A warp walks a contiguous range of token rows; lanes own
// 4-column quads, so the four kinds of column sums (d_norm_w over everything; dgate / dshift / dscale per batch element)
// stay in registers and are flushed with atomics when the batch element changes and at the end.  Every row operand is
// read once as raw 8/16-byte vectors; 22 B read + 10 B written per element (bf16), pure HBM streaming.
constexpr int TAILB_ROWS = 16;

// DET: warps are partitioned per batch element instead -- wpb = nwarps / batch warps per element, warp w takes an equal
// contiguous share of the rows of element w / wpb (warps past batch * wpb idle) -- so that a warp never crosses a batch
// boundary; dgate / dshift / dscale of p address partial rows, one per warp index within the element, (wpb, batch, dim),
// stored (zeros for a warp without rows), not added (zg_block_tail_bwd_det).  d_norm_w is the same partials buffer in both.
// DP (zg_block_tail_bwd_dp): the gradient reaching hidden through the forward's `hidden * path_scale[b]` is
// dh = round(round(dr) * path_scale[b]); d_x, d_mix and dgate follow from that dh, everything else is unchanged.
template <typename T, int MAXQ, bool DET>
__global__ void __launch_bounds__(128, 3) block_tail_bwd_kernel(const zg_block_tail_bwd_params p) {
    constexpr bool DP = false;
    [[maybe_unused]] const void *const path_scale = nullptr;
#include "block_tail_bwd_body.cuh"
}

template <typename T, int MAXQ, bool DET>
__global__ void __launch_bounds__(128, 3) block_tail_dp_bwd_kernel(const zg_block_tail_bwd_dp_params q) {
    constexpr bool DP = true;
    const zg_block_tail_bwd_params &p = q.base;
    const void *const path_scale = q.path_scale;
#include "block_tail_bwd_body.cuh"
}

// path_scale NULL: block_tail_bwd_kernel; otherwise block_tail_dp_bwd_kernel (same MAXQ buckets, grid and shared memory)
template <typename T, bool DET> static int block_tail_bwd_t(const zg_block_tail_bwd_params &p, const void *path_scale, cudaStream_t s) {
    const unsigned grid = (unsigned)p.nparts;          // persistent: the caller sized the d_norm_w partials buffer
    // dynamic shared memory: 4 warps x 3 accumulator sets x MAXQ quads x 32 lanes x 16 B  (<= 48 KB for MAXQ <= 8)
#define ZG_TAILB(Q)                                                                                                             \
    do {                                                                                                                        \
        if (path_scale) block_tail_dp_bwd_kernel<T, Q, DET><<<grid, 128, 4 * 3 * Q * 32 * 16, s>>>(zg_block_tail_bwd_dp_params{p, path_scale}); \
        else block_tail_bwd_kernel<T, Q, DET><<<grid, 128, 4 * 3 * Q * 32 * 16, s>>>(p);                                          \
    } while (0)
    if (p.dim <= 512) ZG_TAILB(4);
    else if (p.dim <= 640) ZG_TAILB(5);
    else if (p.dim <= 768) ZG_TAILB(6);
    else ZG_TAILB(8);
#undef ZG_TAILB
    zg_count_launch();
    return zg_check_launch(path_scale ? "block_tail_bwd_dp" : "block_tail_bwd");
}

// ------------------------------------------------------------------------------------------------
// Text prologue (see include/zigma_b200.h): hidden = x + gate * mix[rowmap], no-affine LayerNorm (norm_msa), modulate.
// The four-warps-per-row layout of block_tail_row4_body: one 128-thread CTA per token row, every operand of the row loaded
// as raw 8/16-byte vectors before the first use, the row kept in registers through the mean, the variance (two-pass, as
// the reference's fp32 LayerNorm statistics) and the output pass.  Reads x, mix; writes hidden, q_in: 4 row passes.
template <typename T, int MAXQ>
__global__ void __launch_bounds__(128, (MAXQ * sizeof(T) <= 4) ? ZG_TAIL_MINB : (MAXQ * sizeof(T) <= 8) ? 8 : 5) text_prologue_fwd_kernel(const zg_text_prologue_params p) {
    __shared__ float red[2][4];
    const int64_t row = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int D = p.dim, nq = D >> 2;
    const int b = (int)(row / p.seqlen), l = (int)(row % p.seqlen);
    const T *x = reinterpret_cast<const T *>(p.x) + row * D;
    const T *mix = reinterpret_cast<const T *>(p.mix) + ((int64_t)b * p.seqlen + (p.rowmap ? p.rowmap[l] : l)) * D;
    const T *gate = reinterpret_cast<const T *>(p.gate) + (int64_t)b * p.mod_rs;
    const T *shift = reinterpret_cast<const T *>(p.shift) + (int64_t)b * p.mod_rs;
    const T *scale = reinterpret_cast<const T *>(p.scale) + (int64_t)b * p.mod_rs;
    T *hidden = reinterpret_cast<T *>(p.hidden) + row * D;
    T *q_in = reinterpret_cast<T *>(p.q_in) + row * D;
    auto block_sum = [&](float v, int slot) {
        v = zg_warp_sum(v);
        if (lane == 0) red[slot][warp] = v;
        __syncthreads();
        return (red[slot][0] + red[slot][1]) + (red[slot][2] + red[slot][3]);
    };
    Raw4<T> rx[MAXQ], rm[MAXQ], rg[MAXQ], rsc[MAXQ], rsh[MAXQ];
#pragma unroll
    for (int k = 0; k < MAXQ; ++k) {
        const int q = tid + 128 * k;
        if (q < nq) {
            rx[k] = ldraw<T>(x, 4 * q);
            rm[k] = ldraw<T>(mix, 4 * q);
            rg[k] = ldraw<T>(gate, 4 * q);
            rsc[k] = ldraw<T>(scale, 4 * q);
            rsh[k] = ldraw<T>(shift, 4 * q);
        }
    }
    float h[MAXQ][4];
    float sum = 0.f;
#pragma unroll
    for (int k = 0; k < MAXQ; ++k) {
        const int q = tid + 128 * k;
        if (q < nq) {
            float m[4], g[4];
            cvt4<T>(rx[k], h[k]);
            cvt4<T>(rm[k], m);
            cvt4<T>(rg[k], g);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                h[k][i] = round_to<T>(h[k][i] + round_to<T>(g[i] * m[i]));
                sum += h[k][i];
            }
            st4<T>(hidden, 4 * q, h[k]);
        }
    }
    const float mean = block_sum(sum, 0) / D;
    float s2 = 0.f;
#pragma unroll
    for (int k = 0; k < MAXQ; ++k)
        if (tid + 128 * k < nq)
#pragma unroll
            for (int i = 0; i < 4; ++i) { const float d = h[k][i] - mean; s2 += d * d; }
    const float rstd = 1.f / sqrtf(block_sum(s2, 1) / D + p.eps);
    if (tid == 0) {
        if (p.mean) p.mean[row] = mean;
        if (p.rstd) p.rstd[row] = rstd;
    }
#pragma unroll
    for (int k = 0; k < MAXQ; ++k) {
        const int q = tid + 128 * k;
        if (q < nq) {
            float sc[4], sh[4], o[4];
            cvt4<T>(rsc[k], sc);
            cvt4<T>(rsh[k], sh);
#pragma unroll
            for (int i = 0; i < 4; ++i)    // modulate(ln, shift, scale) at the eager rounding points
                o[i] = round_to<T>(round_to<T>(round_to<T>((h[k][i] - mean) * rstd) * round_to<T>(1.f + sc[i])) + sh[i]);
            st4<T>(q_in, 4 * q, o);
        }
    }
}

template <typename T> static int text_prologue_fwd_t(const zg_text_prologue_params &p, cudaStream_t s) {
    const unsigned grid = (unsigned)((int64_t)p.batch * p.seqlen);
    if (p.dim <= 512) text_prologue_fwd_kernel<T, 1><<<grid, 128, 0, s>>>(p);
    else if (p.dim <= 1024) text_prologue_fwd_kernel<T, 2><<<grid, 128, 0, s>>>(p);
    else if (p.dim <= 1536) text_prologue_fwd_kernel<T, 3><<<grid, 128, 0, s>>>(p);
    else text_prologue_fwd_kernel<T, 4><<<grid, 128, 0, s>>>(p);
    zg_count_launch();
    return zg_check_launch("text_prologue_fwd");
}

// Backward: the persistent-warp layout and the partition of block_tail_bwd_kernel (block_tail_bwd_body.cuh) -- one warp per
// token row, lanes own 4-column quads, contiguous row ranges (DET: warps partitioned per batch element, partial rows indexed
// by the warp's index within its element), the three per-batch column sums in lane-private shared-memory slots, flushed
// when the batch element changes.  The body is not shared with the tail's: its operands differ in type (hidden in the I/O
// dtype with a saved mean against the tail's fp32 r), in the normalisation (LayerNorm without weight against RMSNorm with
// one) and in the rounding points, and the tail's kernels keep the code they have.
template <typename T, int MAXQ, bool DET>
__global__ void __launch_bounds__(128, 3) text_prologue_bwd_kernel(const zg_text_prologue_bwd_params p) {
    extern __shared__ __align__(16) float tp_smem[];
    float4 *acc_s = reinterpret_cast<float4 *>(tp_smem) + (threadIdx.x >> 5) * (3 * MAXQ * 32) + (threadIdx.x & 31);   // [warp][3][MAXQ][32 lanes]
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int lane = threadIdx.x & 31;
    const int64_t nrows = (int64_t)p.batch * p.seqlen;
    const int64_t per = (nrows + nwarps - 1) / nwarps;
    const int D = p.dim, nq = D >> 2;
    const float invD = 1.f / D;
#pragma unroll
    for (int k = 0; k < MAXQ; ++k)
#pragma unroll
        for (int j = 0; j < 3; ++j) acc_s[(j * MAXQ + k) * 32] = make_float4(0.f, 0.f, 0.f, 0.f);
    auto flush_batch = [&](int b) {
#pragma unroll
        for (int k = 0; k < MAXQ; ++k) {
            const int q = lane + 32 * k;
            if (q < nq) {
                float *dst[3] = {p.dgate, p.dshift, p.dscale};
#pragma unroll
                for (int j = 0; j < 3; ++j) {
                    const float4 v = acc_s[(j * MAXQ + k) * 32];
                    if (DET && dst[j]) {
                        *reinterpret_cast<float4 *>(dst[j] + ((warp % (nwarps / p.batch)) * p.batch + b) * D + 4 * q) = v;
                    } else if (dst[j]) {
                        float *o = dst[j] + (int64_t)b * D + 4 * q;
                        atomicAdd(o, v.x); atomicAdd(o + 1, v.y); atomicAdd(o + 2, v.z); atomicAdd(o + 3, v.w);
                    }
                    acc_s[(j * MAXQ + k) * 32] = make_float4(0.f, 0.f, 0.f, 0.f);
                }
            }
        }
    };
    int64_t row0 = min(warp * per, nrows), row1 = min(row0 + per, nrows);
    if constexpr (DET) {
        const int64_t wpb = nwarps / p.batch, bw = warp / wpb, per_b = (p.seqlen + wpb - 1) / wpb;
        row0 = row1 = nrows;
        if (bw < p.batch) {
            row0 = bw * p.seqlen + min((warp % wpb) * per_b, (int64_t)p.seqlen);
            row1 = bw * p.seqlen + min((warp % wpb + 1) * per_b, (int64_t)p.seqlen);
            if (row0 == row1) flush_batch((int)bw);      // no rows: this warp's partial rows are zeros
        }
    }
    if (row0 >= row1) return;
    int cur_b = (int)(row0 / p.seqlen);
    for (int64_t row = row0; row < row1; ++row) {
        const int b = (int)(row / p.seqlen), l = (int)(row % p.seqlen);
        if (b != cur_b) { flush_batch(cur_b); cur_b = b; }
        const int64_t mrow = (int64_t)b * p.seqlen + (p.rowmap ? p.rowmap[l] : l);
        const T *hid = reinterpret_cast<const T *>(p.hidden) + row * D;
        const T *dq = reinterpret_cast<const T *>(p.d_q) + row * D;
        const T *dhid = p.d_hidden ? reinterpret_cast<const T *>(p.d_hidden) + row * D : nullptr;
        const T *mix = reinterpret_cast<const T *>(p.mix) + mrow * D;
        const T *gate = reinterpret_cast<const T *>(p.gate) + (int64_t)b * p.mod_rs;
        const T *scale = reinterpret_cast<const T *>(p.scale) + (int64_t)b * p.mod_rs;
        const float mean = p.mean[row], rstd = p.rstd[row];
        Raw4<T> rh[MAXQ], rdq[MAXQ], rdh[MAXQ], rmx[MAXQ];
#pragma unroll
        for (int k = 0; k < MAXQ; ++k) {
            const int q = lane + 32 * k;
            if (q < nq) {
                rh[k] = ldraw<T>(hid, 4 * q);
                rdq[k] = ldraw<T>(dq, 4 * q);
                if (dhid) rdh[k] = ldraw<T>(dhid, 4 * q);
                rmx[k] = ldraw<T>(mix, 4 * q);
            }
        }
        // ---- d_ln, dshift / dscale, the two LayerNorm-backward row means ----
        float dl[MAXQ][4];
        float c1 = 0.f, c2 = 0.f;
#pragma unroll
        for (int k = 0; k < MAXQ; ++k) {
            const int q = lane + 32 * k;
            if (q < nq) {
                float hv[4], g[4], sc[4];
                cvt4<T>(rh[k], hv);
                cvt4<T>(rdq[k], g);
                ld4<T>(scale, 4 * q, sc);
                float4 ash = acc_s[(1 * MAXQ + k) * 32], asc = acc_s[(2 * MAXQ + k) * 32];
                float *psh = &ash.x, *psc = &asc.x;
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float xh = (hv[i] - mean) * rstd;
                    dl[k][i] = round_to<T>(g[i] * round_to<T>(1.f + sc[i]));
                    psh[i] += g[i];
                    psc[i] = fmaf(g[i], round_to<T>(xh), psc[i]);      // d_q * ln
                    c1 = fmaf(xh, dl[k][i], c1);
                    c2 += dl[k][i];
                }
                acc_s[(1 * MAXQ + k) * 32] = ash; acc_s[(2 * MAXQ + k) * 32] = asc;
            }
        }
        c1 = zg_warp_sum(c1) * invD;
        c2 = zg_warp_sum(c2) * invD;
        // ---- dh, d_x, d_mix, dgate ----
        T *dx = reinterpret_cast<T *>(p.d_x) + row * D;
        T *dmix = reinterpret_cast<T *>(p.d_mix) + mrow * D;
#pragma unroll
        for (int k = 0; k < MAXQ; ++k) {
            const int q = lane + 32 * k;
            if (q < nq) {
                float hv[4], dh[4], m[4], g[4], o[4];
                cvt4<T>(rh[k], hv);
                if (dhid) cvt4<T>(rdh[k], dh);
                else dh[0] = dh[1] = dh[2] = dh[3] = 0.f;
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float xh = (hv[i] - mean) * rstd;
                    dh[i] = round_to<T>(dh[i] + round_to<T>((dl[k][i] - (xh * c1 + c2)) * rstd));
                }
                st4<T>(dx, 4 * q, dh);
                cvt4<T>(rmx[k], m);
                ld4<T>(gate, 4 * q, g);
                float4 ag = acc_s[(0 * MAXQ + k) * 32];
                float *pg = &ag.x;
#pragma unroll
                for (int i = 0; i < 4; ++i) { o[i] = g[i] * dh[i]; pg[i] = fmaf(dh[i], m[i], pg[i]); }
                acc_s[(0 * MAXQ + k) * 32] = ag;
                st4<T>(dmix, 4 * q, o);
            }
        }
    }
    flush_batch(cur_b);
}

template <typename T, bool DET> static int text_prologue_bwd_t(const zg_text_prologue_bwd_params &p, cudaStream_t s) {
    const unsigned grid = (unsigned)p.nparts;
    // dynamic shared memory: 4 warps x 3 accumulator sets x MAXQ quads x 32 lanes x 16 B  (48 KB at MAXQ 8)
    if (p.dim <= 512) text_prologue_bwd_kernel<T, 4, DET><<<grid, 128, 4 * 3 * 4 * 32 * 16, s>>>(p);
    else if (p.dim <= 640) text_prologue_bwd_kernel<T, 5, DET><<<grid, 128, 4 * 3 * 5 * 32 * 16, s>>>(p);
    else if (p.dim <= 768) text_prologue_bwd_kernel<T, 6, DET><<<grid, 128, 4 * 3 * 6 * 32 * 16, s>>>(p);
    else text_prologue_bwd_kernel<T, 8, DET><<<grid, 128, 4 * 3 * 8 * 32 * 16, s>>>(p);
    zg_count_launch();
    return zg_check_launch("text_prologue_bwd");
}

template <typename T, typename R> static int norm_fwd_tr(const zg_norm_params &p, cudaStream_t s) {
    const int64_t nthreads = (int64_t)p.nrows * 32;
    add_norm_fwd_kernel<T, R><<<(unsigned)((nthreads + 127) / 128), 128, 0, s>>>(p);
    zg_count_launch();
    return zg_check_launch("add_norm_fwd");
}
template <typename T> static int norm_fwd_t(const zg_norm_params &p, cudaStream_t s) {
    if (p.res_dtype == ZG_F32) return norm_fwd_tr<T, float>(p, s);
    if (p.res_dtype == p.dtype) return norm_fwd_tr<T, T>(p, s);
    return zg_set_error("add_norm_fwd: residual dtype must be fp32 or the activation dtype");
}
// launch shape of the backward (host arithmetic only; the launch and the deterministic workspace query share it):
// CTAs (at most 528, whatever the SM count) and whether the vectorised kernel runs
static unsigned norm_bwd_grid(const zg_norm_bwd_params &p) {
    const int64_t want = ((int64_t)p.nrows * 32 + 127) / 128;
    return (unsigned)(want < 132 * 4 ? want : 132 * 4);
}
static bool norm_bwd_vec(const zg_norm_bwd_params &p) {
    const uintptr_t al = reinterpret_cast<uintptr_t>(p.dy) | reinterpret_cast<uintptr_t>(p.x) | reinterpret_cast<uintptr_t>(p.dresidual) |
                         reinterpret_cast<uintptr_t>(p.dx) | reinterpret_cast<uintptr_t>(p.dresidual_in);
    const int64_t so = p.dy_rs | p.x_rs | p.dx_rs | (p.dresidual ? p.dres_rs : 0) | (p.dresidual_in ? p.dresin_rs : 0);
    return p.ncols % 4 == 0 && al % 16 == 0 && so % 4 == 0 && p.ncols <= 1024;
}
template <typename T, typename R, bool DET> static int norm_bwd_tr(const zg_norm_bwd_params &p, cudaStream_t s) {
    const unsigned grid = norm_bwd_grid(p);
    if (norm_bwd_vec(p)) {
        const int nq = p.ncols / 4;
        if (nq <= 32 * 2) add_norm_bwd_vec_kernel<T, R, 2, DET><<<grid, 128, 0, s>>>(p);
        else if (nq <= 32 * 4) add_norm_bwd_vec_kernel<T, R, 4, DET><<<grid, 128, 0, s>>>(p);
        else if (nq <= 32 * 5) add_norm_bwd_vec_kernel<T, R, 5, DET><<<grid, 128, 0, s>>>(p);
        else if (nq <= 32 * 6) add_norm_bwd_vec_kernel<T, R, 6, DET><<<grid, 128, 0, s>>>(p);
        else add_norm_bwd_vec_kernel<T, R, 8, DET><<<grid, 128, 0, s>>>(p);
        zg_count_launch();
        return zg_check_launch("add_norm_bwd(vec)");
    }
    add_norm_bwd_kernel<T, R, DET><<<grid, 128, 0, s>>>(p);
    zg_count_launch();
    return zg_check_launch("add_norm_bwd");
}
template <typename T, bool DET> static int norm_bwd_t(const zg_norm_bwd_params &p, cudaStream_t s) {
    if (p.res_dtype == ZG_F32) return norm_bwd_tr<T, float, DET>(p, s);
    if (p.res_dtype == p.dtype) return norm_bwd_tr<T, T, DET>(p, s);
    return zg_set_error("add_norm_bwd: residual dtype must be fp32 or the activation dtype");
}

}  // namespace zg

static bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
// the block tail reads gate / shift / scale / norm_w as 4-element vectors (ld4 / ldraw): 8 bytes for 16-bit dtypes, 16 for fp32
static bool aligned_quad(const void *p, int dtype) {
    return (reinterpret_cast<uintptr_t>(p) & (4 * (dtype == ZG_F32 ? sizeof(float) : sizeof(__half)) - 1)) == 0;
}

extern "C" int zg_add_norm_fwd(const zg_norm_params *pp, void *stream) {
    ZG_REQUIRE(pp != nullptr, "add_norm_fwd: null params");
    const zg_norm_params &p = *pp;
    ZG_REQUIRE(p.x && p.y, "add_norm_fwd: null tensor pointer");
    ZG_REQUIRE(p.ncols > 0 && p.ncols % 4 == 0 && p.ncols <= 4 * 32 * zg::NORM_MAXQ,
               "add_norm_fwd: ncols must be a multiple of 4 and <= %d, got %d", 4 * 32 * zg::NORM_MAXQ, p.ncols);
    ZG_REQUIRE(p.x_rs % 4 == 0 && p.y_rs % 4 == 0 && p.res_rs % 4 == 0 && p.resout_rs % 4 == 0, "add_norm_fwd: row strides must be multiples of 4");
    ZG_REQUIRE(aligned16(p.x) && aligned16(p.y) && aligned16(p.residual) && aligned16(p.residual_out), "add_norm_fwd: pointers must be 16-byte aligned");
    if (p.nrows == 0) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    switch (p.dtype) {
        case ZG_F32: return zg::norm_fwd_t<float>(p, s);
        case ZG_F16: return zg::norm_fwd_t<__half>(p, s);
        case ZG_BF16: return zg::norm_fwd_t<__nv_bfloat16>(p, s);
    }
    return zg_set_error("add_norm_fwd: bad dtype %d", p.dtype);
}

static int norm_bwd_validate(const zg_norm_bwd_params &p) {
    ZG_REQUIRE(p.dy && p.x && p.dx && p.rstd, "add_norm_bwd: null tensor pointer");
    ZG_REQUIRE(p.ncols > 0 && p.ncols <= 4 * 32 * zg::NORM_MAXQ, "add_norm_bwd: ncols must be <= %d, got %d", 4 * 32 * zg::NORM_MAXQ, p.ncols);
    ZG_REQUIRE(p.dtype == ZG_F32 || p.dtype == ZG_F16 || p.dtype == ZG_BF16, "add_norm_bwd: bad dtype %d", p.dtype);
    return 0;
}

template <bool DET> static int norm_bwd_dispatch(const zg_norm_bwd_params &p, cudaStream_t s) {
    switch (p.dtype) {
        case ZG_F32: return zg::norm_bwd_t<float, DET>(p, s);
        case ZG_F16: return zg::norm_bwd_t<__half, DET>(p, s);
        default: return zg::norm_bwd_t<__nv_bfloat16, DET>(p, s);
    }
}

extern "C" int zg_add_norm_bwd(const zg_norm_bwd_params *pp, void *stream) {
    ZG_REQUIRE(pp != nullptr, "add_norm_bwd: null params");
    if (int rc = norm_bwd_validate(*pp)) return rc;
    if (pp->nrows == 0) return 0;
    return norm_bwd_dispatch<false>(*pp, (cudaStream_t)stream);
}

// partial rows of the deterministic backward: one per CTA (vectorised kernel) or per warp (scalar kernel)
static ZgDetLayout norm_bwd_det_layout(const zg_norm_bwd_params &p, void *ws) {
    ZgDetLayout lay;
    lay.ws = static_cast<unsigned char *>(ws);
    if (p.nrows <= 0 || p.ncols <= 0) return lay;
    const int64_t rows = (int64_t)zg::norm_bwd_grid(p) * (zg::norm_bwd_vec(p) ? 1 : 4);
    lay.add(p.dweight, rows, p.ncols);
    lay.add(p.dbias, rows, p.ncols);
    return lay;
}

extern "C" int64_t zg_add_norm_bwd_det_workspace_bytes(const zg_norm_bwd_params *p) {
    return p ? norm_bwd_det_layout(*p, nullptr).bytes : 0;
}

extern "C" int zg_add_norm_bwd_det(const zg_norm_bwd_params *pp, void *workspace, int64_t workspace_bytes, void *stream) {
    ZG_REQUIRE(pp != nullptr, "add_norm_bwd_det: null params");
    if (int rc = norm_bwd_validate(*pp)) return rc;
    if (pp->nrows == 0) return 0;
    const ZgDetLayout lay = norm_bwd_det_layout(*pp, workspace);
    ZG_REQUIRE_WORKSPACE(lay, workspace, workspace_bytes, "add_norm_bwd_det");
    zg_norm_bwd_params p = *pp;                 // the kernel writes partial rows; the reduction adds them to the outputs
    int i = 0;
    if (p.dweight) p.dweight = lay.reg[i++].part;
    if (p.dbias) p.dbias = lay.reg[i++].part;
    cudaStream_t s = (cudaStream_t)stream;
    if (int rc = norm_bwd_dispatch<true>(p, s)) return rc;
    return lay.reduce(s);
}

static int block_tail_fwd_validate(const zg_block_tail_params &p, bool pe, bool rebuild = false) {
    ZG_REQUIRE((rebuild || (p.x && p.normed)) && p.norm_w, "block_tail_fwd: null tensor pointer");
    if (pe) ZG_REQUIRE(p.mix && !p.gate && !p.rowmap && !p.residual, "block_tail_fwd_pe: takes the (seqlen, dim) table as mix and no gate / rowmap / residual");
    else ZG_REQUIRE(!p.mix || p.gate, "block_tail_fwd: mix needs gate");
    ZG_REQUIRE(!p.modded || (p.shift && p.scale), "block_tail_fwd: modded needs shift and scale");
    ZG_REQUIRE(p.dim > 0 && p.dim % 4 == 0 && p.dim <= 4 * 32 * zg::NORM_MAXQ, "block_tail_fwd: dim must be a multiple of 4 and <= %d, got %d",
               4 * 32 * zg::NORM_MAXQ, p.dim);
    ZG_REQUIRE(p.mod_rs % 4 == 0, "block_tail_fwd: modulation row stride must be a multiple of 4");
    ZG_REQUIRE(aligned16(p.x) && aligned16(p.mix) && aligned16(p.residual) && aligned16(p.residual_out) && aligned16(p.normed) && aligned16(p.modded),
               "block_tail_fwd: row tensors must be 16-byte aligned");
    ZG_REQUIRE(aligned_quad(p.gate, p.dtype) && aligned_quad(p.shift, p.dtype) && aligned_quad(p.scale, p.dtype) && aligned_quad(p.norm_w, p.dtype),
               "block_tail_fwd: gate / shift / scale / norm_w must be aligned to 4 elements");
    return 0;
}

static int block_tail_fwd_entry(const zg_block_tail_params *pp, void *stream, bool pe) {
    ZG_REQUIRE(pp != nullptr, "block_tail_fwd: null params");
    const zg_block_tail_params &p = *pp;
    if (int rc = block_tail_fwd_validate(p, pe)) return rc;
    const int64_t nrows = (int64_t)p.batch * p.seqlen;
    if (nrows == 0) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    switch (p.dtype) {
        case ZG_F32: return zg::block_tail_t<float>(p, s, pe);
        case ZG_F16: return zg::block_tail_t<__half>(p, s, pe);
        case ZG_BF16: return zg::block_tail_t<__nv_bfloat16>(p, s, pe);
    }
    return zg_set_error("block_tail_fwd: bad dtype %d", p.dtype);
}

extern "C" int zg_block_tail_fwd(const zg_block_tail_params *pp, void *stream) { return block_tail_fwd_entry(pp, stream, false); }
extern "C" int zg_block_tail_fwd_pe(const zg_block_tail_params *pp, void *stream) { return block_tail_fwd_entry(pp, stream, true); }

// path_scale is read as one dtype element per batch element
static bool aligned_elem(const void *p, int dtype) {
    return (reinterpret_cast<uintptr_t>(p) & ((dtype == ZG_F32 ? sizeof(float) : sizeof(__half)) - 1)) == 0;
}

extern "C" int zg_block_tail_fwd_rebuild(const zg_block_tail_rebuild_params *pp, void *stream) {
    ZG_REQUIRE(pp != nullptr, "block_tail_fwd_rebuild: null params");
    const zg_block_tail_params &p = pp->base;
    ZG_REQUIRE(p.x == nullptr, "block_tail_fwd_rebuild: x must be NULL (it is rebuilt from residual, x_rstd and x_norm_w)");
    ZG_REQUIRE(p.residual && pp->x_rstd && pp->x_norm_w, "block_tail_fwd_rebuild: needs residual, x_rstd and x_norm_w");
    ZG_REQUIRE(p.normed || !p.final_layer, "block_tail_fwd_rebuild: final_layer needs normed");
    ZG_REQUIRE(p.dim <= 1024, "block_tail_fwd_rebuild: dim must be <= 1024, got %d", p.dim);
    if (int rc = block_tail_fwd_validate(p, false, true)) return rc;
    ZG_REQUIRE(aligned_quad(pp->x_norm_w, p.dtype) && (reinterpret_cast<uintptr_t>(pp->x_rstd) & 3) == 0,
               "block_tail_fwd_rebuild: x_norm_w must be aligned to 4 elements, x_rstd to 4 bytes");
    const int64_t nrows = (int64_t)p.batch * p.seqlen;
    if (nrows == 0) return 0;
    ZG_REQUIRE(nrows <= 0x7fffffffLL, "block_tail_fwd_rebuild: fewer than 2^31 rows only");
    cudaStream_t s = (cudaStream_t)stream;
    switch (p.dtype) {
        case ZG_F32: return zg::block_tail_rebuild_t<float>(*pp, s);
        case ZG_F16: return zg::block_tail_rebuild_t<__half>(*pp, s);
        case ZG_BF16: return zg::block_tail_rebuild_t<__nv_bfloat16>(*pp, s);
    }
    return zg_set_error("block_tail_fwd_rebuild: bad dtype %d", p.dtype);
}

extern "C" int zg_block_tail_fwd_dp(const zg_block_tail_dp_params *pp, void *stream) {
    ZG_REQUIRE(pp != nullptr, "block_tail_fwd_dp: null params");
    const zg_block_tail_params &p = pp->base;
    ZG_REQUIRE(pp->path_scale != nullptr, "block_tail_fwd_dp: null path_scale");
    ZG_REQUIRE(p.residual != nullptr && p.mix != nullptr, "block_tail_fwd_dp: needs residual and mix (the first block has no drop path)");
    ZG_REQUIRE(p.final_layer == 0, "block_tail_fwd_dp: final_layer is not supported");
    ZG_REQUIRE(p.dim <= 1024, "block_tail_fwd_dp: dim must be <= 1024, got %d", p.dim);
    if (int rc = block_tail_fwd_validate(p, false)) return rc;
    ZG_REQUIRE(aligned_elem(pp->path_scale, p.dtype), "block_tail_fwd_dp: path_scale must be aligned to its element size");
    const int64_t nrows = (int64_t)p.batch * p.seqlen;
    if (nrows == 0) return 0;
    ZG_REQUIRE(nrows <= 0x7fffffffLL, "block_tail_fwd_dp: fewer than 2^31 rows only");
    cudaStream_t s = (cudaStream_t)stream;
    switch (p.dtype) {
        case ZG_F32: return zg::block_tail_dp_t<float>(*pp, s);
        case ZG_F16: return zg::block_tail_dp_t<__half>(*pp, s);
        case ZG_BF16: return zg::block_tail_dp_t<__nv_bfloat16>(*pp, s);
    }
    return zg_set_error("block_tail_fwd_dp: bad dtype %d", p.dtype);
}

static int block_tail_bwd_validate(const zg_block_tail_bwd_params &p) {
    ZG_REQUIRE(p.r && p.rstd && p.norm_w && p.d_x, "block_tail_bwd: null tensor pointer");
    ZG_REQUIRE((p.mix != nullptr) == (p.gate != nullptr) && (p.mix != nullptr) == (p.d_mix != nullptr), "block_tail_bwd: mix, gate and d_mix go together");
    ZG_REQUIRE(!p.d_modded || p.scale, "block_tail_bwd: d_modded needs scale");
    ZG_REQUIRE(p.dim > 0 && p.dim % 4 == 0 && p.dim <= 1024, "block_tail_bwd: dim must be a multiple of 4 and <= 1024, got %d", p.dim);
    ZG_REQUIRE(p.mod_rs % 4 == 0, "block_tail_bwd: modulation row stride must be a multiple of 4");
    ZG_REQUIRE(p.nparts >= 1 && p.nparts <= 65535, "block_tail_bwd: nparts (rows of the d_norm_w partials buffer = CTAs) must be in [1, 65535]");
    ZG_REQUIRE(p.dtype == ZG_F32 || p.dtype == ZG_F16 || p.dtype == ZG_BF16, "block_tail_bwd: bad dtype %d", p.dtype);
    ZG_REQUIRE(aligned16(p.r) && aligned16(p.d_residual_out) && aligned16(p.d_normed) && aligned16(p.d_modded) && aligned16(p.mix) && aligned16(p.d_x) &&
                   aligned16(p.d_mix) && aligned16(p.d_residual_in),
               "block_tail_bwd: row tensors must be 16-byte aligned");
    ZG_REQUIRE(aligned_quad(p.gate, p.dtype) && aligned_quad(p.scale, p.dtype) && aligned_quad(p.norm_w, p.dtype),
               "block_tail_bwd: gate / scale / norm_w must be aligned to 4 elements");
    return 0;
}

template <bool DET> static int block_tail_bwd_dispatch(const zg_block_tail_bwd_params &p, const void *path_scale, cudaStream_t s) {
    switch (p.dtype) {
        case ZG_F32: return zg::block_tail_bwd_t<float, DET>(p, path_scale, s);
        case ZG_F16: return zg::block_tail_bwd_t<__half, DET>(p, path_scale, s);
        default: return zg::block_tail_bwd_t<__nv_bfloat16, DET>(p, path_scale, s);
    }
}

extern "C" int zg_block_tail_bwd(const zg_block_tail_bwd_params *pp, void *stream) {
    ZG_REQUIRE(pp != nullptr, "block_tail_bwd: null params");
    if (int rc = block_tail_bwd_validate(*pp)) return rc;
    if (pp->batch == 0 || pp->seqlen == 0) return 0;
    return block_tail_bwd_dispatch<false>(*pp, nullptr, (cudaStream_t)stream);
}

// the drop-path backward takes everything the plain one takes, plus a path_scale; a block without mix has no drop path
static int block_tail_bwd_dp_validate(const zg_block_tail_bwd_dp_params *pp) {
    ZG_REQUIRE(pp != nullptr, "block_tail_bwd_dp: null params");
    ZG_REQUIRE(pp->path_scale != nullptr, "block_tail_bwd_dp: null path_scale");
    ZG_REQUIRE(pp->base.mix != nullptr, "block_tail_bwd_dp: needs mix (the first block has no drop path)");
    if (int rc = block_tail_bwd_validate(pp->base)) return rc;
    ZG_REQUIRE(aligned_elem(pp->path_scale, pp->base.dtype), "block_tail_bwd_dp: path_scale must be aligned to its element size");
    return 0;
}

extern "C" int zg_block_tail_bwd_dp(const zg_block_tail_bwd_dp_params *pp, void *stream) {
    if (int rc = block_tail_bwd_dp_validate(pp)) return rc;
    if (pp->base.batch == 0 || pp->base.seqlen == 0) return 0;
    return block_tail_bwd_dispatch<false>(pp->base, pp->path_scale, (cudaStream_t)stream);
}

// partial rows of the deterministic backward: one per warp index within a batch element (see block_tail_bwd_kernel)
static ZgDetLayout block_tail_bwd_det_layout(const zg_block_tail_bwd_params &p, void *ws) {
    ZgDetLayout lay;
    lay.ws = static_cast<unsigned char *>(ws);
    if (p.batch <= 0 || p.seqlen <= 0 || p.dim <= 0 || p.nparts < 1) return lay;
    const int64_t wpb = 4 * (int64_t)p.nparts / p.batch, n = (int64_t)p.batch * p.dim;
    lay.add(p.dgate, wpb, n);
    lay.add(p.dshift, wpb, n);
    lay.add(p.dscale, wpb, n);
    return lay;
}

extern "C" int64_t zg_block_tail_bwd_det_workspace_bytes(const zg_block_tail_bwd_params *p) {
    return p ? block_tail_bwd_det_layout(*p, nullptr).bytes : 0;
}

// validated params; path_scale NULL for the plain entry point
static int block_tail_bwd_det_run(const zg_block_tail_bwd_params &q, const void *path_scale, void *workspace, int64_t workspace_bytes, void *stream) {
    if (q.batch == 0 || q.seqlen == 0) return 0;
    ZG_REQUIRE(4 * (int64_t)q.nparts >= q.batch, "block_tail_bwd_det: needs at least one warp per batch element (4 * nparts >= batch), got nparts %d for batch %d",
               q.nparts, q.batch);
    const ZgDetLayout lay = block_tail_bwd_det_layout(q, workspace);
    ZG_REQUIRE_WORKSPACE(lay, workspace, workspace_bytes, "block_tail_bwd_det");
    zg_block_tail_bwd_params p = q;             // the kernel writes partial rows; the reduction adds them to the outputs
    int i = 0;
    if (p.dgate) p.dgate = lay.reg[i++].part;
    if (p.dshift) p.dshift = lay.reg[i++].part;
    if (p.dscale) p.dscale = lay.reg[i++].part;
    cudaStream_t s = (cudaStream_t)stream;
    if (int rc = block_tail_bwd_dispatch<true>(p, path_scale, s)) return rc;
    return lay.reduce(s);
}

extern "C" int zg_block_tail_bwd_det(const zg_block_tail_bwd_params *pp, void *workspace, int64_t workspace_bytes, void *stream) {
    ZG_REQUIRE(pp != nullptr, "block_tail_bwd_det: null params");
    if (int rc = block_tail_bwd_validate(*pp)) return rc;
    return block_tail_bwd_det_run(*pp, nullptr, workspace, workspace_bytes, stream);
}

// the multiplier does not touch any column sum's layout: the same partials as the plain deterministic backward
extern "C" int64_t zg_block_tail_bwd_dp_det_workspace_bytes(const zg_block_tail_bwd_dp_params *p) {
    return p ? block_tail_bwd_det_layout(p->base, nullptr).bytes : 0;
}

extern "C" int zg_block_tail_bwd_dp_det(const zg_block_tail_bwd_dp_params *pp, void *workspace, int64_t workspace_bytes, void *stream) {
    if (int rc = block_tail_bwd_dp_validate(pp)) return rc;
    return block_tail_bwd_det_run(pp->base, pp->path_scale, workspace, workspace_bytes, stream);
}

static int text_prologue_fwd_validate(const zg_text_prologue_params &p) {
    ZG_REQUIRE(p.x && p.mix && p.gate && p.shift && p.scale && p.hidden && p.q_in, "text_prologue_fwd: null tensor pointer");
    ZG_REQUIRE(p.batch >= 0 && p.seqlen >= 0, "text_prologue_fwd: negative batch or seqlen");
    ZG_REQUIRE(p.dim > 0 && p.dim % 4 == 0 && p.dim <= 4 * 32 * zg::NORM_MAXQ, "text_prologue_fwd: dim must be a multiple of 4 and <= %d, got %d",
               4 * 32 * zg::NORM_MAXQ, p.dim);
    ZG_REQUIRE(p.mod_rs % 4 == 0, "text_prologue_fwd: modulation row stride must be a multiple of 4");
    ZG_REQUIRE(p.dtype == ZG_F32 || p.dtype == ZG_F16 || p.dtype == ZG_BF16, "text_prologue_fwd: bad dtype %d", p.dtype);
    ZG_REQUIRE(aligned16(p.x) && aligned16(p.mix) && aligned16(p.hidden) && aligned16(p.q_in), "text_prologue_fwd: row tensors must be 16-byte aligned");
    ZG_REQUIRE(aligned_quad(p.gate, p.dtype) && aligned_quad(p.shift, p.dtype) && aligned_quad(p.scale, p.dtype),
               "text_prologue_fwd: gate / shift / scale must be aligned to 4 elements");
    ZG_REQUIRE((int64_t)p.batch * p.seqlen <= 0x7fffffffLL, "text_prologue_fwd: fewer than 2^31 rows only");
    return 0;
}

extern "C" int zg_text_prologue_fwd(const zg_text_prologue_params *pp, void *stream) {
    ZG_REQUIRE(pp != nullptr, "text_prologue_fwd: null params");
    const zg_text_prologue_params &p = *pp;
    if (int rc = text_prologue_fwd_validate(p)) return rc;
    if (p.batch == 0 || p.seqlen == 0) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    switch (p.dtype) {
        case ZG_F32: return zg::text_prologue_fwd_t<float>(p, s);
        case ZG_F16: return zg::text_prologue_fwd_t<__half>(p, s);
        default: return zg::text_prologue_fwd_t<__nv_bfloat16>(p, s);
    }
}

static int text_prologue_bwd_validate(const zg_text_prologue_bwd_params &p) {
    ZG_REQUIRE(p.d_q && p.hidden && p.mix && p.gate && p.scale && p.mean && p.rstd && p.d_x && p.d_mix, "text_prologue_bwd: null tensor pointer");
    ZG_REQUIRE(p.batch >= 0 && p.seqlen >= 0, "text_prologue_bwd: negative batch or seqlen");
    ZG_REQUIRE(p.dim > 0 && p.dim % 4 == 0 && p.dim <= 1024, "text_prologue_bwd: dim must be a multiple of 4 and <= 1024, got %d", p.dim);
    ZG_REQUIRE(p.mod_rs % 4 == 0, "text_prologue_bwd: modulation row stride must be a multiple of 4");
    ZG_REQUIRE(p.nparts >= 1 && p.nparts <= 65535, "text_prologue_bwd: nparts (CTAs) must be in [1, 65535]");
    ZG_REQUIRE(p.dtype == ZG_F32 || p.dtype == ZG_F16 || p.dtype == ZG_BF16, "text_prologue_bwd: bad dtype %d", p.dtype);
    ZG_REQUIRE(aligned16(p.d_hidden) && aligned16(p.d_q) && aligned16(p.hidden) && aligned16(p.mix) && aligned16(p.d_x) && aligned16(p.d_mix),
               "text_prologue_bwd: row tensors must be 16-byte aligned");
    ZG_REQUIRE(aligned_quad(p.gate, p.dtype) && aligned_quad(p.scale, p.dtype), "text_prologue_bwd: gate / scale must be aligned to 4 elements");
    return 0;
}

template <bool DET> static int text_prologue_bwd_dispatch(const zg_text_prologue_bwd_params &p, cudaStream_t s) {
    switch (p.dtype) {
        case ZG_F32: return zg::text_prologue_bwd_t<float, DET>(p, s);
        case ZG_F16: return zg::text_prologue_bwd_t<__half, DET>(p, s);
        default: return zg::text_prologue_bwd_t<__nv_bfloat16, DET>(p, s);
    }
}

extern "C" int zg_text_prologue_bwd(const zg_text_prologue_bwd_params *pp, void *stream) {
    ZG_REQUIRE(pp != nullptr, "text_prologue_bwd: null params");
    if (int rc = text_prologue_bwd_validate(*pp)) return rc;
    if (pp->batch == 0 || pp->seqlen == 0) return 0;
    return text_prologue_bwd_dispatch<false>(*pp, (cudaStream_t)stream);
}

// partial rows of the deterministic backward: one per warp index within a batch element (the block tail's layout)
static ZgDetLayout text_prologue_bwd_det_layout(const zg_text_prologue_bwd_params &p, void *ws) {
    ZgDetLayout lay;
    lay.ws = static_cast<unsigned char *>(ws);
    if (p.batch <= 0 || p.seqlen <= 0 || p.dim <= 0 || p.nparts < 1) return lay;
    const int64_t wpb = 4 * (int64_t)p.nparts / p.batch, n = (int64_t)p.batch * p.dim;
    lay.add(p.dgate, wpb, n);
    lay.add(p.dshift, wpb, n);
    lay.add(p.dscale, wpb, n);
    return lay;
}

extern "C" int64_t zg_text_prologue_bwd_det_workspace_bytes(const zg_text_prologue_bwd_params *p) {
    return p ? text_prologue_bwd_det_layout(*p, nullptr).bytes : 0;
}

extern "C" int zg_text_prologue_bwd_det(const zg_text_prologue_bwd_params *pp, void *workspace, int64_t workspace_bytes, void *stream) {
    ZG_REQUIRE(pp != nullptr, "text_prologue_bwd_det: null params");
    if (int rc = text_prologue_bwd_validate(*pp)) return rc;
    if (pp->batch == 0 || pp->seqlen == 0) return 0;
    ZG_REQUIRE(4 * (int64_t)pp->nparts >= pp->batch, "text_prologue_bwd_det: needs at least one warp per batch element (4 * nparts >= batch), got nparts %d for batch %d",
               pp->nparts, pp->batch);
    const ZgDetLayout lay = text_prologue_bwd_det_layout(*pp, workspace);
    ZG_REQUIRE_WORKSPACE(lay, workspace, workspace_bytes, "text_prologue_bwd_det");
    zg_text_prologue_bwd_params p = *pp;        // the kernel writes partial rows; the reduction adds them to the outputs
    int i = 0;
    if (p.dgate) p.dgate = lay.reg[i++].part;
    if (p.dshift) p.dshift = lay.reg[i++].part;
    if (p.dscale) p.dscale = lay.reg[i++].part;
    cudaStream_t s = (cudaStream_t)stream;
    if (int rc = text_prologue_bwd_dispatch<true>(p, s)) return rc;
    return lay.reduce(s);
}
