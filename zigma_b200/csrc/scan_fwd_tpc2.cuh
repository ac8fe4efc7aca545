// Selective-scan forward, hot-path specialisation: token-major (dim-contiguous) activations, N = 16 states,
// input-dependent B/C, everything 16-byte aligned, seqlen a multiple of 16 -- the shape class of every ZigMa
// sampling config.  Same algorithm, staging and numerics as zg::scan_fwd_kernel (scan_fwd.cuh), but TWO
// threads share a channel: each owns 8 of the 16 states (4 fp32x2 pairs) and half of the per-step scalar
// work (softplus of one step, SiLU gate + store of one step, exchanged with one SHFL each way).
//
// Why: with one thread per channel the kernel needs 96 registers per thread and the grid (B*E/32 = 2560 warps
// at BASELINE config 2) only supplies 4.3 warps per SM sub-partition; a profile of it showed
// the scheduler with ~1.1 eligible warps per cycle and `wait` (fixed-latency dependency) as the top stall.
// Splitting the states halves the live registers (<= 56) and doubles the resident warps (8.6 per SMSP) for the
// same total instruction and MUFU count, so the MUFU pipe -- the real bound of this kernel -- stays fed.
//
// Tried and rejected (an earlier experiment): a warp-autonomous variant (every warp stages / converts / consumes its own
// 8-step tiles, __syncwarp instead of the three block barriers per 16 steps) -- bit-identical results, 0.638 ms instead of
// 0.557 ms: the extra per-warp staging work and the 4x B/C traffic cost more than the barriers do.
#pragma once
#include "scan_fwd.cuh"

namespace zg {

constexpr int TPC2_THREADS = 128;   // 64 channels x 2 threads

template <typename T, bool CKPT = false>
__global__ void __launch_bounds__(TPC2_THREADS, 9) scan_fwd_tpc2_kernel(const zg_scan_params p) {
    static_assert(sizeof(T) == 2, "16-bit I/O only");
    constexpr int NS = 16, CH = SCAN_CH, TL = SCAN_TL, NSTAGE = 3, VEC = 8;
    constexpr int ACT_BYTES = TL * CH * 2;                  // one tensor, one stage: [TL][CH] of T
    constexpr int RAW_BC = TL * NS * 2;                     // [TL][NS] of T
    constexpr int STAGE = 3 * ACT_BYTES + 2 * RAW_BC;
    extern __shared__ __align__(16) unsigned char smem[];
    float *bcf = reinterpret_cast<float *>(smem + NSTAGE * STAGE);     // [TL][B0..15 C0..15] fp32

    const int tid = threadIdx.x;
    const int c = tid >> 1, hf = tid & 1;
    const int E = p.dim, L = p.seqlen;
    const int per_group = E / p.ngroups;
    const int tiles_per_group = per_group / CH;
    const int tiles = tiles_per_group * p.ngroups;
    const int b = blockIdx.x / tiles;
    const int tile = blockIdx.x % tiles;
    const int g = tile / tiles_per_group;
    const int e0 = g * per_group + (tile % tiles_per_group) * CH;
    const int e = e0 + c;
    const bool has_z = p.z != nullptr;
    const bool softplus = (p.flags & ZG_SCAN_DELTA_SOFTPLUS) != 0;

    const T *gu = reinterpret_cast<const T *>(p.u) + (int64_t)b * p.u_sb + e0;
    const T *gd = reinterpret_cast<const T *>(p.delta) + (int64_t)b * p.delta_sb + e0;
    const T *gz = has_z ? reinterpret_cast<const T *>(p.z) + (int64_t)b * p.z_sb + e0 : nullptr;
    const T *gB = reinterpret_cast<const T *>(p.B) + (int64_t)b * p.B_sb + (int64_t)g * p.B_sg;
    const T *gC = reinterpret_cast<const T *>(p.C) + (int64_t)b * p.C_sb + (int64_t)g * p.C_sg;
    T *gout = reinterpret_cast<T *>(p.out) + (int64_t)b * p.out_sb + e;

    zg_f2 Al2p[4], h2[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int n = 8 * hf + 2 * q;
        Al2p[q].x = p.A[(int64_t)e * NS + n] * ZG_LOG2E;
        Al2p[q].y = p.A[(int64_t)e * NS + n + 1] * ZG_LOG2E;
        h2[q] = zg_splat2(0.f);
    }
    const float Dv = p.D ? p.D[e] : 0.f;
    const float bias = p.delta_bias ? p.delta_bias[e] : 0.f;
    const int nstages = L / TL;

    auto issue_stage = [&](int s) {
        if (s < nstages) {
            unsigned char *st = smem + (s % NSTAGE) * STAGE;
            const int l0 = s * TL;
            // 16 steps x 8 chunks of 16 bytes = 128 chunks per tensor = one per thread
            const int t = tid >> 3, j = tid & 7;
            const int l = l0 + t;
            unsigned char *dst = st + t * (CH * 2) + j * 16;
            // in-batch offsets fit 32 bits (checked on the host): one IMAD each instead of 64-bit multiplies
            zg_cp_async16(dst, gu + (l * (int)p.u_sl + j * VEC));
            zg_cp_async16(dst + ACT_BYTES, gd + (l * (int)p.delta_sl + j * VEC));
            if (has_z) zg_cp_async16(dst + 2 * ACT_BYTES, gz + ((p.z_rowmap ? p.z_rowmap[l] : l) * (int)p.z_sl + j * VEC));
            if (tid < 64) {                                 // B, C rows: 2 x 16 steps x 2 chunks
                const int w = tid >> 5, t = (tid >> 1) & 15, j = tid & 1;
                const T *src = (w ? gC + (l0 + t) * (int)p.C_sl : gB + (l0 + t) * (int)p.B_sl) + j * VEC;
                zg_cp_async16(st + 3 * ACT_BYTES + w * RAW_BC + t * (NS * 2) + j * 16, src);
            }
        }
        zg_cp_async_commit();
    };

#pragma unroll
    for (int s = 0; s < NSTAGE - 1; ++s) issue_stage(s);

    for (int s = 0; s < nstages; ++s) {
        issue_stage(s + NSTAGE - 1);
        zg_cp_async_wait<NSTAGE - 1>();
        __syncthreads();
        unsigned char *st = smem + (s % NSTAGE) * STAGE;
        if (tid < 64) {     // raw B/C -> fp32, one 16-byte chunk (8 states of one step) per thread
            const int w = tid >> 5, t = (tid >> 1) & 15, j = tid & 1;
            union { uint4 v; T e[8]; } R;
            R.v = *reinterpret_cast<const uint4 *>(st + 3 * ACT_BYTES + w * RAW_BC + t * (NS * 2) + j * 16);
            float4 o0, o1;
            o0.x = zg_to_float<T>(R.e[0]); o0.y = zg_to_float<T>(R.e[1]); o0.z = zg_to_float<T>(R.e[2]); o0.w = zg_to_float<T>(R.e[3]);
            o1.x = zg_to_float<T>(R.e[4]); o1.y = zg_to_float<T>(R.e[5]); o1.z = zg_to_float<T>(R.e[6]); o1.w = zg_to_float<T>(R.e[7]);
            float4 *d4 = reinterpret_cast<float4 *>(bcf + t * 2 * NS + w * NS + j * 8);
            d4[0] = o0; d4[1] = o1;
        }
        __syncthreads();

        const T *su = reinterpret_cast<const T *>(st) + c;
        const T *sd = reinterpret_cast<const T *>(st + ACT_BYTES) + c;
        const T *sz = reinterpret_cast<const T *>(st + 2 * ACT_BYTES) + c;
        T *ocol = gout + (s * TL) * (int)p.out_sl;
#pragma unroll 1
        for (int t0 = 0; t0 < TL; t0 += 2) {
            // scalars: this thread owns step t0 + hf (softplus, gate, store); delta' crosses with one SHFL
            const int tm = t0 + hf;
            const float u0 = zg_to_float<T>(su[t0 * CH]), u1 = zg_to_float<T>(su[(t0 + 1) * CH]);
            float dm = zg_to_float<T>(sd[tm * CH]) + bias;
            if (softplus) dm = zg_softplus20(dm);
            const float dother = __shfl_xor_sync(0xffffffffu, dm, 1);
            const float d0 = hf ? dother : dm, d1 = hf ? dm : dother;
            const zg_f2 dl2[2] = {zg_splat2(d0), zg_splat2(d1)};
            const zg_f2 du2[2] = {zg_splat2(d0 * u0), zg_splat2(d1 * u1)};
            zg_f2 y2[2] = {zg_splat2(0.f), zg_splat2(0.f)};
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const float4 *bc = reinterpret_cast<const float4 *>(bcf + (t0 + i) * 2 * NS + 8 * hf);
                const float4 B0 = bc[0], B1 = bc[1], C0 = bc[4], C1 = bc[5];
                const zg_f2 Bp[4] = {make_float2(B0.x, B0.y), make_float2(B0.z, B0.w), make_float2(B1.x, B1.y), make_float2(B1.z, B1.w)};
                const zg_f2 Cp[4] = {make_float2(C0.x, C0.y), make_float2(C0.z, C0.w), make_float2(C1.x, C1.y), make_float2(C1.z, C1.w)};
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const zg_f2 x = zg_mul2(dl2[i], Al2p[q]);
                    const zg_f2 a = zg_ex2_mufu2(x);
                    h2[q] = zg_fma2(a, h2[q], zg_mul2(du2[i], Bp[q]));
                    y2[i] = zg_fma2(Cp[q], h2[q], y2[i]);
                }
            }
            const float yp0 = y2[0].x + y2[0].y, yp1 = y2[1].x + y2[1].y;
            // partner finalises the other step: hand it our partial sum of that step, take its partial of ours
            const float recv = __shfl_xor_sync(0xffffffffu, hf ? yp0 : yp1, 1);
            float y = (hf ? yp1 : yp0) + recv + Dv * (hf ? u1 : u0);
            if (has_z) y *= zg_silu(zg_to_float<T>(sz[tm * CH]));
            ocol[tm * (int)p.out_sl] = zg_from_float<T>(y);
            if (CKPT && ((t0 + 2) & 7) == 0) {   // (compile-time: the sampling instantiation carries no trace of it; host side: ckpt_every == 8)       // recompute seeds for the backward pass: every 8 steps (uniform branch)
                // (batch, n_ckpt, dim, dstate): the 16 channels x 2 halves of a warp write 1 KB contiguous
                float4 *dst = reinterpret_cast<float4 *>(p.ckpt + (((int64_t)b * (L >> 3) + ((s * TL + t0 + 2) >> 3) - 1) * E + e) * NS + 8 * hf);
                dst[0] = make_float4(h2[0].x, h2[0].y, h2[1].x, h2[1].y);
                dst[1] = make_float4(h2[2].x, h2[2].y, h2[3].x, h2[3].y);
            }
        }
        __syncthreads();
    }
    if (p.last_state) {
        float *dst = p.last_state + ((int64_t)b * E + e) * NS + 8 * hf;
#pragma unroll
        for (int q = 0; q < 4; ++q) { dst[2 * q] = h2[q].x; dst[2 * q + 1] = h2[q].y; }
    }
}

// host-side eligibility test + launch; returns -1 when the call does not fit the specialisation
template <typename T> int try_launch_scan_fwd_tpc2(const zg_scan_params &p, cudaStream_t stream) {
    static int enabled = -1;
    if (enabled < 0) { const char *e = getenv("ZG_SCAN_TPC2"); enabled = e ? atoi(e) : 1; }
    if (!enabled || sizeof(T) != 2) return -1;
    const bool varBC = (p.flags & ZG_SCAN_VARIABLE_B) && (p.flags & ZG_SCAN_VARIABLE_C);
    if (!varBC || p.dstate != 16 || p.seqlen % SCAN_TL != 0 || p.seqlen == 0) return -1;
    if (p.ckpt && p.ckpt_every != 8) return -1;
    if ((p.dim / p.ngroups) % SCAN_CH != 0) return -1;
    if (!(p.u_sd == 1 && p.delta_sd == 1 && p.out_sd == 1 && (!p.z || p.z_sd == 1) && p.B_sn == 1 && p.C_sn == 1)) return -1;
    const uintptr_t al = reinterpret_cast<uintptr_t>(p.u) | reinterpret_cast<uintptr_t>(p.delta) | reinterpret_cast<uintptr_t>(p.z) |
                         reinterpret_cast<uintptr_t>(p.B) | reinterpret_cast<uintptr_t>(p.C);
    const int64_t so = p.u_sb | p.delta_sb | (p.z ? p.z_sb : 0) | p.B_sb | p.B_sg | p.C_sb | p.C_sg | p.u_sl | p.delta_sl | (p.z ? p.z_sl : 0) | p.B_sl | p.C_sl;
    if (al % 16 != 0 || so % 8 != 0 || reinterpret_cast<uintptr_t>(p.ckpt) % 16 != 0) return -1;
    // 32-bit in-batch offsets inside the kernel
    const int64_t lim = 0x7fffffffLL;
    if ((int64_t)p.seqlen * p.u_sl > lim || (int64_t)p.seqlen * p.delta_sl > lim || (p.z && (int64_t)p.seqlen * p.z_sl > lim) ||
        (int64_t)p.seqlen * p.out_sl > lim || (int64_t)p.seqlen * p.B_sl > lim || (int64_t)p.seqlen * p.C_sl > lim)
        return -1;
    constexpr int smem = 3 * (3 * SCAN_TL * SCAN_CH * 2 + 2 * SCAN_TL * 16 * 2) + SCAN_TL * 32 * 4;
    const long long nblk = (long long)(p.dim / SCAN_CH) * p.batch;
    if (nblk > 0x7fffffffLL) return -1;
    auto launch = [&](auto kern) {
        static bool attr_set = false;
        if (!attr_set) {
            cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
            cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
            attr_set = true;
        }
        kern<<<(unsigned)nblk, TPC2_THREADS, smem, stream>>>(p);
    };
    if (p.ckpt) launch(scan_fwd_tpc2_kernel<T, true>);          // training forward (writes the recompute seeds)
    else launch(scan_fwd_tpc2_kernel<T>);
    zg_count_launch();
    zg_note_scan_kernel("zg::scan_fwd_tpc2_kernel (round 1: LDGSTS ring, two threads per channel)");
    return zg_check_launch("scan_fwd(tpc2)");
}

}  // namespace zg
