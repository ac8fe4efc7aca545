// Text cross-attention of has_text blocks (zg_cross_attn_fwd / _bwd, include/zigma_b200.h; DESIGN.md section 4.7):
//     O = softmax(Q K^T * 0.125) V      per (batch, head), head dimension 64, 1 <= Lk <= 256 keys, no mask, no dropout
// Q, O (batch, L, heads * 64) and K, V (batch, Lk, heads * 64) are read and written token-major through row strides, so
// the (B, H, L, 64) copies of the library path are not needed.
//
// Kernels:
//   xattn_fwd_mma_kernel<T>   16-bit forward on the tensor cores (mma.sync m16n8k16): one CTA per (four 64-query tiles,
//                             head, batch), K and V of the head in shared memory, each warp owns 16 query rows of a tile;
//                             keys in chunks of 64 with online rescaling of the running max.
//   xattn_rows_kernel<T, BWD> one warp per query row on the CUDA cores: the fp32 forward (BWD = false) and, for every dtype,
//                             the dQ part of the backward (BWD = true), which also writes D_i = sum dO_i * O_i.
//   xattn_bwd_kv_kernel<T>    dK / dV partial sums of one segment of query rows for 32 keys, stored (no atomics) in the
//                             segment's own slice of the workspace;
//   xattn_bwd_reduce_kernel<T> adds the segments in index order and writes dK, dV in the I/O dtype.
#include "zg_common.cuh"
#include <type_traits>

namespace zg {

constexpr int XA_HD = 64;              // head dimension
constexpr int XA_MAX_KEYS = 256;
constexpr float XA_SCALE = 0.125f;     // 1 / sqrt(64)
constexpr int XA_KS = XA_HD + 1;       // fp32 smem row stride of the CUDA-core kernels (conflict-free column walks)
constexpr int XA_MS = XA_HD + 8;       // 16-bit smem row stride of the MMA kernel: 144-byte rows, conflict-free ldmatrix
constexpr int XA_ROWS_WARPS = 8;       // warps of xattn_rows_kernel
constexpr int XA_ROWS_PER_CTA = 128;   // query rows per CTA of xattn_rows_kernel (K, V staged once for all of them)
constexpr int XA_MMA_TILES = 4;        // 64-query tiles per CTA of xattn_fwd_mma_kernel (K, V staged once for all of them)
constexpr int XA_KV_KEYS = 32;         // keys per CTA of xattn_bwd_kv_kernel
constexpr int XA_KV_TILE = 32;         // query rows staged per step of xattn_bwd_kv_kernel
constexpr int XA_SEG_ROWS = 64;        // a backward segment is a whole number of 64-row query tiles

struct XattnArgs {
    const void *q, *k, *v, *o, *dout;
    void *out;                         // forward: O; backward: dQ
    float *lse;                        // (batch, heads, L): forward output (optional) / backward input
    float *dvec;                       // backward: D (batch, heads, L)
    int64_t q_sb, q_rs, k_sb, k_rs, v_sb, v_rs, o_sb, o_rs, do_sb, do_rs, out_sb, out_rs;
    int batch, L, Lk, heads;
};

// 2^x keeping subnormal results (ex2.approx without .ftz): a probability below 2^-126 still counts in fp32 gradients
__device__ __forceinline__ float xa_ex2(float x) {
    float y;
    asm("ex2.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// 8 consecutive values (16 bytes) of a row, as fp32
template <typename T> __device__ __forceinline__ void xa_load8(const T *p, float *f);
template <> __device__ __forceinline__ void xa_load8<float>(const float *p, float *f) {
    const float4 a = *reinterpret_cast<const float4 *>(p), b = *reinterpret_cast<const float4 *>(p + 4);
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
template <typename T> __device__ __forceinline__ void xa_load8(const T *p, float *f) {
    const uint4 r = *reinterpret_cast<const uint4 *>(p);
    const T *h = reinterpret_cast<const T *>(&r);
#pragma unroll
    for (int i = 0; i < 8; ++i) f[i] = zg_to_float<T>(h[i]);
}

// rows [0, n) of one head (64 columns at `src`, row stride rs) -> fp32 shared rows of stride XA_KS
template <typename T>
__device__ __forceinline__ void xa_stage_f32(float *dst, const T *src, int64_t rs, int n) {
    for (int i = threadIdx.x; i < n * (XA_HD / 8); i += blockDim.x) {
        const int r = i >> 3, c = (i & 7) * 8;
        float f[8];
        xa_load8<T>(src + r * rs + c, f);
#pragma unroll
        for (int e = 0; e < 8; ++e) dst[r * XA_KS + c + e] = f[e];
    }
}

// ================================================================================================================
// 16-bit forward, tensor cores
// ================================================================================================================
template <typename T> __device__ __forceinline__ uint32_t xa_pack(float lo, float hi);
template <> __device__ __forceinline__ uint32_t xa_pack<__half>(float lo, float hi) {
    __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t *>(&h);
}
template <> __device__ __forceinline__ uint32_t xa_pack<__nv_bfloat16>(float lo, float hi) {
    __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t *>(&h);
}

template <typename T>
__device__ __forceinline__ void xa_mma(float *c, const uint32_t *a, uint32_t b0, uint32_t b1) {
    if constexpr (std::is_same<T, __half>::value) {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    } else {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    }
}

__device__ __forceinline__ void xa_ldmatrix_x4_trans(uint32_t *r, const void *smem) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(zg_smem_u32(smem)));
}

// Per warp, rows r0 = lane/4 and r1 = r0 + 8 of its 16: S = Q K^T in fp32 accumulators, scores scaled into the log2 domain,
// running max m and running sum l in fp32; P = 2^(s - m) rounded to T as the A operand of P V; O accumulated in fp32 and
// divided by l once; one rounding at the store.
template <typename T>
__global__ void __launch_bounds__(128) xattn_fwd_mma_kernel(const XattnArgs a) {
    extern __shared__ __align__(16) unsigned char xa_smem[];
    T *sK = reinterpret_cast<T *>(xa_smem);
    const int Lk = a.Lk, Lkp = (Lk + 15) & ~15;
    T *sV = sK + Lkp * XA_MS;
    const int b = blockIdx.z, h = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const T *K = static_cast<const T *>(a.k) + b * a.k_sb + h * XA_HD;
    const T *V = static_cast<const T *>(a.v) + b * a.v_sb + h * XA_HD;
    for (int i = threadIdx.x; i < Lkp * 8; i += blockDim.x) {
        const int r = i >> 3, c = (i & 7) * 8;
        if (r < Lk) {
            zg_cp_async16(sK + r * XA_MS + c, K + r * a.k_rs + c);
            zg_cp_async16(sV + r * XA_MS + c, V + r * a.v_rs + c);
        } else {                       // padded keys: zero K and V rows (their scores are masked to -inf below)
            *reinterpret_cast<uint4 *>(sK + r * XA_MS + c) = make_uint4(0, 0, 0, 0);
            *reinterpret_cast<uint4 *>(sV + r * XA_MS + c) = make_uint4(0, 0, 0, 0);
        }
    }
    zg_cp_async_commit();
    zg_cp_async_wait<0>();
    __syncthreads();
    for (int tile = blockIdx.x * XA_MMA_TILES; tile < (int)(blockIdx.x + 1) * XA_MMA_TILES; ++tile) {
        const int row0 = tile * 64 + warp * 16, r0 = row0 + (lane >> 2), r1 = r0 + 8;
        if (row0 >= a.L) break;
        const int cq = (lane & 3) * 2;
        const T *Q = static_cast<const T *>(a.q) + b * a.q_sb + h * XA_HD;
        uint32_t qa[4][4];                 // A fragments of the warp's 16 x 64 Q tile, 4 k-steps of 16
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            const int c = ks * 16 + cq;
            qa[ks][0] = r0 < a.L ? *reinterpret_cast<const uint32_t *>(Q + r0 * a.q_rs + c) : 0u;
            qa[ks][1] = r1 < a.L ? *reinterpret_cast<const uint32_t *>(Q + r1 * a.q_rs + c) : 0u;
            qa[ks][2] = r0 < a.L ? *reinterpret_cast<const uint32_t *>(Q + r0 * a.q_rs + c + 8) : 0u;
            qa[ks][3] = r1 < a.L ? *reinterpret_cast<const uint32_t *>(Q + r1 * a.q_rs + c + 8) : 0u;
        }

        const float sc = XA_SCALE * ZG_LOG2E;
        float acc[8][4];
#pragma unroll
        for (int n = 0; n < 8; ++n) acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.f;
        float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

        for (int c0 = 0; c0 < Lkp; c0 += 64) {
            const int nt = min(64, Lkp - c0) >> 3;     // 8-key tiles in this chunk (even: Lkp is a multiple of 16)
            float s[8][4];
#pragma unroll
            for (int t = 0; t < 8; ++t) {
                s[t][0] = s[t][1] = s[t][2] = s[t][3] = 0.f;
                if (t < nt) {
                    const T *kr = sK + (c0 + t * 8 + (lane >> 2)) * XA_MS + cq;
#pragma unroll
                    for (int ks = 0; ks < 4; ++ks) {
                        const uint32_t b0 = *reinterpret_cast<const uint32_t *>(kr + ks * 16);
                        const uint32_t b1 = *reinterpret_cast<const uint32_t *>(kr + ks * 16 + 8);
                        xa_mma<T>(s[t], qa[ks], b0, b1);
                    }
                }
            }
            float cm0 = -INFINITY, cm1 = -INFINITY;
#pragma unroll
            for (int t = 0; t < 8; ++t) {
                const int key = c0 + t * 8 + cq;
                const bool ok0 = t < nt && key < Lk, ok1 = t < nt && key + 1 < Lk;
                s[t][0] = ok0 ? s[t][0] * sc : -INFINITY;
                s[t][1] = ok1 ? s[t][1] * sc : -INFINITY;
                s[t][2] = ok0 ? s[t][2] * sc : -INFINITY;
                s[t][3] = ok1 ? s[t][3] * sc : -INFINITY;
                cm0 = fmaxf(cm0, fmaxf(s[t][0], s[t][1]));
                cm1 = fmaxf(cm1, fmaxf(s[t][2], s[t][3]));
            }
#pragma unroll
            for (int o = 1; o <= 2; o <<= 1) {
                cm0 = fmaxf(cm0, __shfl_xor_sync(0xffffffffu, cm0, o));
                cm1 = fmaxf(cm1, __shfl_xor_sync(0xffffffffu, cm1, o));
            }
            // every chunk holds at least one real key, so the new max is finite (for finite scores)
            const float mn0 = fmaxf(m0, cm0), mn1 = fmaxf(m1, cm1);
            const float al0 = xa_ex2(m0 - mn0), al1 = xa_ex2(m1 - mn1);   // 0 on the first chunk (m = -inf)
            m0 = mn0; m1 = mn1;
            float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
            for (int t = 0; t < 8; ++t) {
                s[t][0] = xa_ex2(s[t][0] - m0);
                s[t][1] = xa_ex2(s[t][1] - m0);
                s[t][2] = xa_ex2(s[t][2] - m1);
                s[t][3] = xa_ex2(s[t][3] - m1);
                ps0 += s[t][0] + s[t][1];
                ps1 += s[t][2] + s[t][3];
            }
            l0 = l0 * al0 + ps0;
            l1 = l1 * al1 + ps1;
#pragma unroll
            for (int n = 0; n < 8; ++n) {
                acc[n][0] *= al0; acc[n][1] *= al0;
                acc[n][2] *= al1; acc[n][3] *= al1;
            }
            // O += P V: k-step j covers keys c0 + 16 j .. + 15; the S accumulators of tiles 2j, 2j+1 are its A fragment
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (2 * j < nt) {
                    uint32_t pa[4];
                    pa[0] = xa_pack<T>(s[2 * j][0], s[2 * j][1]);
                    pa[1] = xa_pack<T>(s[2 * j][2], s[2 * j][3]);
                    pa[2] = xa_pack<T>(s[2 * j + 1][0], s[2 * j + 1][1]);
                    pa[3] = xa_pack<T>(s[2 * j + 1][2], s[2 * j + 1][3]);
                    // lane l addresses row (key) c0 + 16 j + (l % 8) + 8 ((l / 8) % 2), columns 8 (l / 16) .. of each 16-dim pair
                    const T *vr = sV + (c0 + 16 * j + (lane & 7) + ((lane >> 3) & 1) * 8) * XA_MS + (lane >> 4) * 8;
#pragma unroll
                    for (int n2 = 0; n2 < 4; ++n2) {
                        uint32_t vb[4];
                        xa_ldmatrix_x4_trans(vb, vr + n2 * 16);
                        xa_mma<T>(acc[2 * n2], pa, vb[0], vb[1]);
                        xa_mma<T>(acc[2 * n2 + 1], pa, vb[2], vb[3]);
                    }
                }
            }
        }
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {
            l0 += __shfl_xor_sync(0xffffffffu, l0, o);
            l1 += __shfl_xor_sync(0xffffffffu, l1, o);
        }
        const float inv0 = 1.f / l0, inv1 = 1.f / l1;
        T *O = static_cast<T *>(a.out) + b * a.o_sb + h * XA_HD;
#pragma unroll
        for (int n = 0; n < 8; ++n) {
            const int c = n * 8 + cq;
            if (r0 < a.L) *reinterpret_cast<uint32_t *>(O + r0 * a.o_rs + c) = xa_pack<T>(acc[n][0] * inv0, acc[n][1] * inv0);
            if (r1 < a.L) *reinterpret_cast<uint32_t *>(O + r1 * a.o_rs + c) = xa_pack<T>(acc[n][2] * inv1, acc[n][3] * inv1);
        }
        if (a.lse != nullptr && (lane & 3) == 0) {
            float *lse = a.lse + ((int64_t)b * a.heads + h) * a.L;
            if (r0 < a.L) lse[r0] = (m0 + __log2f(l0)) * ZG_LN2;
            if (r1 < a.L) lse[r1] = (m1 + __log2f(l1)) * ZG_LN2;
        }
    }
}

// Dot product of two 64-vectors as four sequential 16-term FMA chains added pairwise, the order in which the dK / dV kernel
// forms it across its four lanes per key.  D_i = dO_i.O_i and dO_i.v_j then round identically, so dS = P (dO.v - D) is
// exactly 0 where O_i equals v_j bit for bit (a single key), and so are dQ and dK.
__device__ __forceinline__ float xa_dot64(const float *x, const float *y) {
    float p[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        p[q] = 0.f;
#pragma unroll
        for (int e = 0; e < 16; ++e) p[q] = fmaf(x[q * 16 + e], y[q * 16 + e], p[q]);
    }
    return (p[0] + p[1]) + (p[2] + p[3]);
}

// ================================================================================================================
// CUDA-core row kernel: fp32 forward (BWD = false) and dQ + D of the backward (BWD = true), one warp per query row
// ================================================================================================================
// forward:  s_j = 0.125 log2e q.k_j,  m = max s,  p_j = 2^(s_j - m),  o = sum_j p_j v_j / sum_j p_j,  lse = (m + log2 l) ln2
// backward: D = dO.O,  p_j = 2^(0.125 log2e q.k_j - lse log2e),  ds_j = p_j (dO.v_j - D),  dq = 0.125 sum_j ds_j k_j
template <typename T, bool BWD>
__global__ void __launch_bounds__(256) xattn_rows_kernel(const XattnArgs a) {
    extern __shared__ __align__(16) float xa_fsmem[];
    const int Lk = a.Lk;
    float *sK = xa_fsmem, *sV = sK + Lk * XA_KS;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float *sq = sV + Lk * XA_KS + warp * (3 * XA_HD + XA_MAX_KEYS);   // per warp: q, dO, O, p / ds
    float *sdo = sq + XA_HD, *so = sdo + XA_HD, *sp = so + XA_HD;
    const int b = blockIdx.z, h = blockIdx.y;
    xa_stage_f32<T>(sK, static_cast<const T *>(a.k) + b * a.k_sb + h * XA_HD, a.k_rs, Lk);
    xa_stage_f32<T>(sV, static_cast<const T *>(a.v) + b * a.v_sb + h * XA_HD, a.v_rs, Lk);
    __syncthreads();
    const float sc = XA_SCALE * ZG_LOG2E;
    const int64_t bh = (int64_t)b * a.heads + h;
    const int rend = min(a.L, (int)(blockIdx.x + 1) * XA_ROWS_PER_CTA);
    for (int i = blockIdx.x * XA_ROWS_PER_CTA + warp; i < rend; i += XA_ROWS_WARPS) {
        const T *qr = static_cast<const T *>(a.q) + b * a.q_sb + i * a.q_rs + h * XA_HD;
        sq[lane] = zg_to_float<T>(qr[lane]);
        sq[lane + 32] = zg_to_float<T>(qr[lane + 32]);
        float dvec = 0.f, lse2 = 0.f;
        if constexpr (BWD) {
            const T *dor = static_cast<const T *>(a.dout) + b * a.do_sb + i * a.do_rs + h * XA_HD;
            const T *orow = static_cast<const T *>(a.o) + b * a.o_sb + i * a.o_rs + h * XA_HD;
            sdo[lane] = zg_to_float<T>(dor[lane]);
            sdo[lane + 32] = zg_to_float<T>(dor[lane + 32]);
            so[lane] = zg_to_float<T>(orow[lane]);
            so[lane + 32] = zg_to_float<T>(orow[lane + 32]);
            lse2 = a.lse[bh * a.L + i] * ZG_LOG2E;
        }
        __syncwarp();
        if constexpr (BWD) {
            dvec = xa_dot64(sdo, so);
            if (lane == 0) a.dvec[bh * a.L + i] = dvec;
        }
        float mx = -INFINITY;
        for (int j = lane; j < Lk; j += 32) {
            float s = xa_dot64(sq, sK + j * XA_KS);
            if constexpr (BWD) {
                const float dp = xa_dot64(sdo, sV + j * XA_KS);
                sp[j] = xa_ex2(s * sc - lse2) * (dp - dvec);
            } else {
                s *= sc;
                sp[j] = s;
                mx = fmaxf(mx, s);
            }
        }
        float inv = 1.f, l = 0.f;
        if constexpr (!BWD) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
            for (int j = lane; j < Lk; j += 32) {
                const float p = xa_ex2(sp[j] - mx);
                sp[j] = p;
                l += p;
            }
            l = zg_warp_sum(l);
            inv = 1.f / l;
        }
        __syncwarp();
        const float *src = BWD ? sK : sV;                // dq = sum ds_j k_j;  o = sum p_j v_j
        float o0 = 0.f, o1 = 0.f;
        for (int j = 0; j < Lk; ++j) {
            const float w = sp[j];
            o0 = fmaf(w, src[j * XA_KS + lane], o0);
            o1 = fmaf(w, src[j * XA_KS + lane + 32], o1);
        }
        const float f = BWD ? XA_SCALE : inv;
        T *outr = static_cast<T *>(a.out) + b * a.out_sb + i * a.out_rs + h * XA_HD;
        outr[lane] = zg_from_float<T>(o0 * f);
        outr[lane + 32] = zg_from_float<T>(o1 * f);
        if constexpr (!BWD) {
            if (a.lse != nullptr && lane == 0) a.lse[bh * a.L + i] = (mx + __log2f(l)) * ZG_LN2;
        }
        __syncwarp();
    }
}

// ================================================================================================================
// dK / dV partials: CTA = (32 keys, one segment of query rows, batch * head); thread = (key, 16 of the 64 dims)
// ================================================================================================================
template <typename T>
__global__ void __launch_bounds__(128) xattn_bwd_kv_kernel(const XattnArgs a, int seg_rows, float *__restrict__ part) {
    constexpr int RS = 80, PS = 20;                    // staged row stride / per-quarter offset (conflict-free float4 reads)
    __shared__ __align__(16) float sq[XA_KV_TILE * RS], sdo[XA_KV_TILE * RS];
    __shared__ float slse[XA_KV_TILE], sdv[XA_KV_TILE];
    const int bh = blockIdx.z, b = bh / a.heads, h = bh % a.heads, seg = blockIdx.y;
    const int quarter = threadIdx.x & 3, key = blockIdx.x * XA_KV_KEYS + (threadIdx.x >> 2);
    const bool kok = key < a.Lk;
    float kf[16], vf[16], dk[16], dv[16];
    {
        const int kk = kok ? key : 0;
        const T *kr = static_cast<const T *>(a.k) + b * a.k_sb + kk * a.k_rs + h * XA_HD + quarter * 16;
        const T *vr = static_cast<const T *>(a.v) + b * a.v_sb + kk * a.v_rs + h * XA_HD + quarter * 16;
        xa_load8<T>(kr, kf);
        xa_load8<T>(kr + 8, kf + 8);
        xa_load8<T>(vr, vf);
        xa_load8<T>(vr + 8, vf + 8);
    }
#pragma unroll
    for (int e = 0; e < 16; ++e) dk[e] = dv[e] = 0.f;
    const float sc = XA_SCALE * ZG_LOG2E;
    const int rbeg = seg * seg_rows, rend = min(a.L, rbeg + seg_rows);
    for (int t0 = rbeg; t0 < rend; t0 += XA_KV_TILE) {
        const int nr = min(XA_KV_TILE, rend - t0);
        __syncthreads();
        for (int i = threadIdx.x; i < nr * 8; i += blockDim.x) {
            const int r = i >> 3, c = (i & 7) * 8, dst = r * RS + (c >> 4) * PS + (c & 15);
            float f[8];
            xa_load8<T>(static_cast<const T *>(a.q) + b * a.q_sb + (t0 + r) * a.q_rs + h * XA_HD + c, f);
#pragma unroll
            for (int e = 0; e < 8; ++e) sq[dst + e] = f[e];
            xa_load8<T>(static_cast<const T *>(a.dout) + b * a.do_sb + (t0 + r) * a.do_rs + h * XA_HD + c, f);
#pragma unroll
            for (int e = 0; e < 8; ++e) sdo[dst + e] = f[e];
        }
        if (threadIdx.x < nr) {
            slse[threadIdx.x] = a.lse[(int64_t)bh * a.L + t0 + threadIdx.x] * ZG_LOG2E;
            sdv[threadIdx.x] = a.dvec[(int64_t)bh * a.L + t0 + threadIdx.x];
        }
        __syncthreads();
        for (int r = 0; r < nr; ++r) {
            const float4 *q4 = reinterpret_cast<const float4 *>(sq + r * RS + quarter * PS);
            const float4 *d4 = reinterpret_cast<const float4 *>(sdo + r * RS + quarter * PS);
            float qv[16], dov[16];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float4 x = q4[e], y = d4[e];
                qv[4 * e] = x.x; qv[4 * e + 1] = x.y; qv[4 * e + 2] = x.z; qv[4 * e + 3] = x.w;
                dov[4 * e] = y.x; dov[4 * e + 1] = y.y; dov[4 * e + 2] = y.z; dov[4 * e + 3] = y.w;
            }
            float s = 0.f, dp = 0.f;
#pragma unroll
            for (int e = 0; e < 16; ++e) {
                s = fmaf(qv[e], kf[e], s);
                dp = fmaf(dov[e], vf[e], dp);
            }
            s += __shfl_xor_sync(0xffffffffu, s, 1);
            dp += __shfl_xor_sync(0xffffffffu, dp, 1);
            s += __shfl_xor_sync(0xffffffffu, s, 2);
            dp += __shfl_xor_sync(0xffffffffu, dp, 2);
            const float p = xa_ex2(s * sc - slse[r]);
            const float ds = p * (dp - sdv[r]);
#pragma unroll
            for (int e = 0; e < 16; ++e) {
                dv[e] = fmaf(p, dov[e], dv[e]);
                dk[e] = fmaf(ds, qv[e], dk[e]);
            }
        }
    }
    if (!kok) return;
    // partials: [segment][batch * head][key][64] fp32, dK region then dV region
    const int64_t per = (int64_t)gridDim.y * gridDim.z * a.Lk * XA_HD;
    float *pk = part + (((int64_t)seg * gridDim.z + bh) * a.Lk + key) * XA_HD + quarter * 16;
#pragma unroll
    for (int e = 0; e < 16; e += 4) {
        *reinterpret_cast<float4 *>(pk + e) = make_float4(dk[e], dk[e + 1], dk[e + 2], dk[e + 3]);
        *reinterpret_cast<float4 *>(pk + per + e) = make_float4(dv[e], dv[e + 1], dv[e + 2], dv[e + 3]);
    }
}

// dK = 0.125 sum_seg part_k,  dV = sum_seg part_v, segments added in index order; one thread per output element
template <typename T>
__global__ void __launch_bounds__(256) xattn_bwd_reduce_kernel(const float *__restrict__ part, int nseg, int batch, int heads, int Lk,
                                                              T *dk, int64_t dk_sb, int64_t dk_rs, T *dv, int64_t dv_sb, int64_t dv_rs) {
    const int64_t n = (int64_t)batch * heads * Lk * XA_HD, per = n;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        float sk = 0.f, sv = 0.f;
        for (int s = 0; s < nseg; ++s) {
            sk += part[s * per + i];
            sv += part[((int64_t)nseg + s) * per + i];
        }
        const int d = (int)(i % XA_HD);
        const int64_t r = i / XA_HD;
        const int key = (int)(r % Lk);
        const int64_t bh = r / Lk;
        const int h = (int)(bh % heads), b = (int)(bh / heads);
        dk[b * dk_sb + key * dk_rs + h * XA_HD + d] = zg_from_float<T>(sk * XA_SCALE);
        dv[b * dv_sb + key * dv_rs + h * XA_HD + d] = zg_from_float<T>(sv);
    }
}

// ================================================================================================================
// host side
// ================================================================================================================
static int xa_check(const zg_xattn_params &p, const char *who) {
    ZG_REQUIRE(p.dtype == ZG_F32 || p.dtype == ZG_F16 || p.dtype == ZG_BF16, "%s: bad dtype %d", who, p.dtype);
    ZG_REQUIRE(p.batch >= 0 && p.L >= 0 && p.heads >= 1, "%s: bad shape (batch %d, L %d, heads %d)", who, p.batch, p.L, p.heads);
    ZG_REQUIRE(p.Lk >= 1 && p.Lk <= XA_MAX_KEYS, "%s: Lk must be in [1, %d], got %d", who, XA_MAX_KEYS, p.Lk);
    ZG_REQUIRE(p.dim % XA_HD == 0, "%s: inner width %d is not a multiple of %d", who, p.dim, XA_HD);
    ZG_REQUIRE(p.dim == XA_HD * p.heads, "%s: inner width %d != %d heads x head dimension %d", who, p.dim, p.heads, XA_HD);
    ZG_REQUIRE(p.q && p.k && p.v && p.o, "%s: null tensor pointer", who);
    return 0;
}

// 16-byte base pointers and row / batch strides that are whole multiples of 16 bytes (the vector and cp.async loads)
static bool xa_aligned(const void *ptr, int64_t sb, int64_t rs, int esz) {
    const int64_t v = 16 / esz;
    return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0 && sb % v == 0 && rs % v == 0;
}

#define XA_REQUIRE_ALIGNED(ptr, sb, rs, esz, who, name)                                                           \
    ZG_REQUIRE(xa_aligned(ptr, sb, rs, esz), "%s: %s must be 16-byte aligned with batch / row strides of whole 16 bytes", \
               who, name)

static int xa_segments(int batch, int heads, int L, int Lk, int sms, int *seg_rows) {
    // about two waves of 4 CTAs per SM for the dK / dV kernel, each segment a whole number of 64-row query tiles
    const int64_t tiles = (L + XA_SEG_ROWS - 1) / XA_SEG_ROWS;
    const int64_t ctas = (int64_t)batch * heads * ((Lk + XA_KV_KEYS - 1) / XA_KV_KEYS);
    const int64_t want = (8LL * (sms > 0 ? sms : 1) + ctas - 1) / ctas;
    const int64_t nseg0 = want < tiles ? want : tiles;
    const int64_t per = (tiles + nseg0 - 1) / nseg0;
    *seg_rows = (int)(per * XA_SEG_ROWS);
    return (int)((tiles + per - 1) / per);
}

static int64_t xa_ws_bytes(const zg_xattn_bwd_params &p, int *nseg, int *seg_rows) {
    const zg_xattn_params &f = p.fwd;
    if (f.batch <= 0 || f.L <= 0 || f.heads <= 0 || f.Lk <= 0) {
        *nseg = 0;
        *seg_rows = 0;
        return 0;
    }
    *nseg = xa_segments(f.batch, f.heads, f.L, f.Lk, p.sms, seg_rows);
    const int64_t dbytes = ((int64_t)f.batch * f.heads * f.L * 4 + 15) / 16 * 16;
    return dbytes + 2LL * *nseg * f.batch * f.heads * f.Lk * XA_HD * 4;
}

static XattnArgs xa_args(const zg_xattn_params &p) {
    XattnArgs a{};
    a.q = p.q; a.k = p.k; a.v = p.v; a.o = p.o;
    a.lse = p.lse;
    a.q_sb = p.q_sb; a.q_rs = p.q_rs; a.k_sb = p.k_sb; a.k_rs = p.k_rs;
    a.v_sb = p.v_sb; a.v_rs = p.v_rs; a.o_sb = p.o_sb; a.o_rs = p.o_rs;
    a.batch = p.batch; a.L = p.L; a.Lk = p.Lk; a.heads = p.heads;
    return a;
}

static size_t xa_rows_smem(int Lk) { return ((size_t)2 * Lk * XA_KS + XA_ROWS_WARPS * (3 * XA_HD + XA_MAX_KEYS)) * sizeof(float); }

template <typename T, bool BWD>
static int xa_launch_rows(const XattnArgs &a, cudaStream_t s) {
    const size_t smem = xa_rows_smem(a.Lk);
    cudaFuncSetAttribute(xattn_rows_kernel<T, BWD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const dim3 grid((a.L + XA_ROWS_PER_CTA - 1) / XA_ROWS_PER_CTA, a.heads, a.batch);
    xattn_rows_kernel<T, BWD><<<grid, XA_ROWS_WARPS * 32, smem, s>>>(a);
    zg_count_launch();
    return zg_check_launch(BWD ? "cross_attn_bwd (dq)" : "cross_attn_fwd (fp32)");
}

template <typename T>
static int xa_launch_fwd_mma(const XattnArgs &a, cudaStream_t s) {
    const size_t smem = (size_t)2 * ((a.Lk + 15) & ~15) * XA_MS * sizeof(T);
    cudaFuncSetAttribute(xattn_fwd_mma_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const dim3 grid((a.L + 64 * XA_MMA_TILES - 1) / (64 * XA_MMA_TILES), a.heads, a.batch);
    xattn_fwd_mma_kernel<T><<<grid, 128, smem, s>>>(a);
    zg_count_launch();
    return zg_check_launch("cross_attn_fwd");
}

template <typename T>
static int xa_launch_bwd(const XattnArgs &a, const zg_xattn_bwd_params &p, float *part, int nseg, int seg_rows, cudaStream_t s) {
    if (int rc = xa_launch_rows<T, true>(a, s)) return rc;
    const dim3 grid((a.Lk + XA_KV_KEYS - 1) / XA_KV_KEYS, nseg, a.batch * a.heads);
    xattn_bwd_kv_kernel<T><<<grid, 128, 0, s>>>(a, seg_rows, part);
    zg_count_launch();
    if (int rc = zg_check_launch("cross_attn_bwd (dk, dv)")) return rc;
    const int64_t n = (int64_t)a.batch * a.heads * a.Lk * XA_HD;
    const int64_t want = (n + 255) / 256;
    xattn_bwd_reduce_kernel<T><<<(unsigned)(want < 132 * 16 ? want : 132 * 16), 256, 0, s>>>(
        part, nseg, a.batch, a.heads, a.Lk, static_cast<T *>(p.dk), p.dk_sb, p.dk_rs, static_cast<T *>(p.dv), p.dv_sb, p.dv_rs);
    zg_count_launch();
    return zg_check_launch("cross_attn_bwd (reduce)");
}

}  // namespace zg

extern "C" {

int zg_cross_attn_fwd(const zg_xattn_params *pp, void *stream) {
    using namespace zg;
    static const char *who = "cross_attn_fwd";
    ZG_REQUIRE(pp != nullptr, "%s: null params", who);
    const zg_xattn_params &p = *pp;
    if (int rc = xa_check(p, who)) return rc;
    const int esz = zg_dtype_size(p.dtype);
    XA_REQUIRE_ALIGNED(p.q, p.q_sb, p.q_rs, esz, who, "q");
    XA_REQUIRE_ALIGNED(p.k, p.k_sb, p.k_rs, esz, who, "k");
    XA_REQUIRE_ALIGNED(p.v, p.v_sb, p.v_rs, esz, who, "v");
    XA_REQUIRE_ALIGNED(p.o, p.o_sb, p.o_rs, esz, who, "o");
    if (p.batch == 0 || p.L == 0) return 0;
    ZG_REQUIRE(p.batch <= 65535 && p.heads <= 65535, "%s: batch %d / heads %d above 65535", who, p.batch, p.heads);
    XattnArgs a = xa_args(p);
    a.out = p.o;
    a.out_sb = p.o_sb;
    a.out_rs = p.o_rs;
    cudaStream_t s = (cudaStream_t)stream;
    switch (p.dtype) {
        case ZG_F32: return xa_launch_rows<float, false>(a, s);
        case ZG_F16: return xa_launch_fwd_mma<__half>(a, s);
        default: return xa_launch_fwd_mma<__nv_bfloat16>(a, s);
    }
}

int64_t zg_cross_attn_bwd_workspace_bytes(const zg_xattn_bwd_params *p) {
    if (p == nullptr) return 0;
    int nseg, seg_rows;
    return zg::xa_ws_bytes(*p, &nseg, &seg_rows);
}

int zg_cross_attn_bwd(const zg_xattn_bwd_params *pp, void *workspace, int64_t workspace_bytes, void *stream) {
    using namespace zg;
    static const char *who = "cross_attn_bwd";
    ZG_REQUIRE(pp != nullptr, "%s: null params", who);
    const zg_xattn_bwd_params &p = *pp;
    const zg_xattn_params &f = p.fwd;
    if (int rc = xa_check(f, who)) return rc;
    ZG_REQUIRE(f.lse && p.dout && p.dq && p.dk && p.dv, "%s: null tensor pointer (lse, dout, dq, dk, dv are required)", who);
    ZG_REQUIRE(p.sms >= 1, "%s: sms must be >= 1, got %d", who, p.sms);
    const int esz = zg_dtype_size(f.dtype);
    XA_REQUIRE_ALIGNED(f.q, f.q_sb, f.q_rs, esz, who, "q");
    XA_REQUIRE_ALIGNED(f.k, f.k_sb, f.k_rs, esz, who, "k");
    XA_REQUIRE_ALIGNED(f.v, f.v_sb, f.v_rs, esz, who, "v");
    XA_REQUIRE_ALIGNED(f.o, f.o_sb, f.o_rs, esz, who, "o");
    XA_REQUIRE_ALIGNED(p.dout, p.dout_sb, p.dout_rs, esz, who, "dout");
    XA_REQUIRE_ALIGNED(p.dq, p.dq_sb, p.dq_rs, esz, who, "dq");
    XA_REQUIRE_ALIGNED(p.dk, p.dk_sb, p.dk_rs, esz, who, "dk");
    XA_REQUIRE_ALIGNED(p.dv, p.dv_sb, p.dv_rs, esz, who, "dv");
    int nseg, seg_rows;
    const int64_t need = xa_ws_bytes(p, &nseg, &seg_rows);
    ZG_REQUIRE(need <= workspace_bytes && (need == 0 || (workspace != nullptr && (reinterpret_cast<uintptr_t>(workspace) & 15) == 0)),
               "%s: workspace of %lld bytes (16-byte aligned) needed, got %lld", who, (long long)need, (long long)workspace_bytes);
    if (f.batch == 0 || f.L == 0) return 0;
    ZG_REQUIRE(f.batch <= 65535 && f.heads <= 65535 && (int64_t)f.batch * f.heads <= 65535,
               "%s: batch %d x heads %d above 65535", who, f.batch, f.heads);
    XattnArgs a = xa_args(f);
    a.dout = p.dout;
    a.do_sb = p.dout_sb;
    a.do_rs = p.dout_rs;
    a.out = p.dq;
    a.out_sb = p.dq_sb;
    a.out_rs = p.dq_rs;
    unsigned char *ws = static_cast<unsigned char *>(workspace);
    a.dvec = reinterpret_cast<float *>(ws);
    float *part = reinterpret_cast<float *>(ws + ((int64_t)f.batch * f.heads * f.L * 4 + 15) / 16 * 16);
    cudaStream_t s = (cudaStream_t)stream;
    switch (f.dtype) {
        case ZG_F32: return xa_launch_bwd<float>(a, p, part, nseg, seg_rows, s);
        case ZG_F16: return xa_launch_bwd<__half>(a, p, part, nseg, seg_rows, s);
        default: return xa_launch_bwd<__nv_bfloat16>(a, p, part, nseg, seg_rows, s);
    }
}

}  // extern "C"
