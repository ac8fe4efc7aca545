// Selective-scan (S6) forward for sm_90a -- sequential-in-L, parallel over (batch, channel, state).
//
// Replaces selective_scan_fwd_kernel (dis_mamba/csrc/selective_scan/selective_scan_fwd_kernel.cuh:67-303).
// The reference maps one CTA to one (batch, channel) row and runs a CUB block scan over L for each
// of the N states in turn (17.4 issued SASS instructions per (b,d,l,n) update, 3 BAR.SYNC per state
// iteration, SURVEY.md section 8a).  At the batch sizes of the sampling path there are B*E >= 80k
// independent recurrences -- more than enough to fill 132 SMs without parallelising over L -- so here
// every THREAD owns one channel, keeps its N states in registers and walks L sequentially:
// 1 FMUL + 1 MUFU.EX2 + 1 FMUL + 2 FFMA per state update, no block-wide scan, no shuffles.
// The (u, delta, z) tiles and the B/C rows of the next steps are staged into shared memory by a
// cp.async (LDGSTS) ring so HBM latency never sits on the recurrence's dependency chain.
//
// Two tile loaders behind one kernel body:
//   SEQ = true   activations (batch, dim, seqlen) with seqlen contiguous -- the reference layout of
//                selective_scan_fn; a thread reads 16-byte vectors along its own row (smem rows
//                padded to an odd number of 16-byte units -> conflict-free LDS.128).
//   SEQ = false  activations (batch, seqlen, dim) with dim contiguous -- the token-major layout of
//                the fused model path; a warp reads 32 consecutive channels of one token (coalesced),
//                B/C come straight from x_dbl rows, and the z half can be gathered through z_rowmap
//                (the zigzag permutation) so no permuted copy of xz is ever materialised.
#pragma once
#include "zg_common.cuh"
#include <stdlib.h>

namespace zg {

constexpr int SCAN_CH = 64;      // channels (= threads) per CTA
constexpr int SCAN_TL = 16;      // time steps per pipeline stage
#ifndef ZG_SCAN_NPOLY_DEFAULT
#define ZG_SCAN_NPOLY_DEFAULT 0
#endif
constexpr int SCAN_SB = 4;       // time steps processed together by the packed inner loop
// The register file is split per SMSP (16384 x 32-bit each): 5 warps per SMSP need <= 96 registers per
// thread.  At bs=64, E=1280 the grid has 2560 warps = 17.3 per SM; with 4 warps per SMSP (100+
// registers) only 16 fit and a second, 8%-full wave doubles the kernel time (ncu round 1:
// launch__waves_per_multiprocessor 1.08).  Asking for 10 CTAs of 64 threads caps ptxas at 96.
constexpr int SCAN_MIN_CTAS = 10;

template <typename T, bool SEQ> struct ScanSmem {
    static constexpr int VEC = 16 / sizeof(T);
    static constexpr int NSTAGE = SEQ ? 2 : 3;
    // SEQ: row = TL elements + one 16-byte pad;  !SEQ: row = CH elements
    static constexpr int ACT_ROW_BYTES = SEQ ? (SCAN_TL * (int)sizeof(T) + 16) : (SCAN_CH * (int)sizeof(T));
    static constexpr int ACT_ROWS = SEQ ? SCAN_CH : SCAN_TL;
    static constexpr int ACT_BYTES = ACT_ROW_BYTES * ACT_ROWS;   // one tensor, one stage
    static __host__ __device__ constexpr int raw_bc_bytes(int NS) { return NS * SCAN_TL * (int)sizeof(T); }
    static __host__ __device__ constexpr int stage_bytes(int NS) { return 3 * ACT_BYTES + 2 * raw_bc_bytes(NS); }
    static __host__ __device__ constexpr int total_bytes(int NS) {
        return NSTAGE * stage_bytes(NS) + SCAN_TL * 2 * NS * (int)sizeof(float);
    }
};

// copy one 16-byte chunk (VEC elements) global -> shared; nvalid = how many leading elements exist
template <typename T>
__device__ __forceinline__ void copy_chunk(T *sdst, const T *gsrc, int nvalid) {
    constexpr int VEC = 16 / sizeof(T);
    if (nvalid >= VEC && ((reinterpret_cast<uintptr_t>(gsrc) & 15) == 0)) {
        zg_cp_async16(sdst, gsrc);
    } else {
#pragma unroll
        for (int i = 0; i < VEC; ++i) sdst[i] = (i < nvalid) ? gsrc[i] : zg_from_float<T>(0.f);
    }
}

// NPOLY: how many of the NS/2 state PAIRS take their exp2 from the FMA-pipe polynomial instead of MUFU
template <typename T, int NS, bool SEQ, bool CONSTBC, int NPOLY>
__global__ void __launch_bounds__(SCAN_CH, (NS <= 16 && !CONSTBC) ? SCAN_MIN_CTAS : 1) scan_fwd_kernel(const zg_scan_params p) {
    using SM = ScanSmem<T, SEQ>;
    constexpr int VEC = SM::VEC;
    constexpr int TL = SCAN_TL, CH = SCAN_CH, NSTAGE = SM::NSTAGE, SB = SCAN_SB, NP = NS / 2;
    extern __shared__ __align__(16) unsigned char smem[];
    float *bcf = reinterpret_cast<float *>(smem + NSTAGE * SM::stage_bytes(NS));   // [TL][2*NS]

    const int tid = threadIdx.x;
    const int E = p.dim, L = p.seqlen, N = p.dstate;
    const int per_group = E / p.ngroups;
    const int tiles_per_group = (per_group + CH - 1) / CH;
    const int tiles = tiles_per_group * p.ngroups;
    const int b = blockIdx.x / tiles;           // 1-D grid: batch may exceed 65535 (video temporal scans)
    const int tile = blockIdx.x % tiles;
    const int g = tile / tiles_per_group;
    const int e0 = g * per_group + (tile % tiles_per_group) * CH;
    const int e_end = min(e0 + CH, (g + 1) * per_group);
    const int e = e0 + tid;
    const bool active = e < e_end;
    const bool has_z = p.z != nullptr;
    const bool softplus = (p.flags & ZG_SCAN_DELTA_SOFTPLUS) != 0;
    const bool varB = (p.flags & ZG_SCAN_VARIABLE_B) != 0;
    const bool varC = (p.flags & ZG_SCAN_VARIABLE_C) != 0;

    const T *gu = reinterpret_cast<const T *>(p.u) + (int64_t)b * p.u_sb;
    const T *gd = reinterpret_cast<const T *>(p.delta) + (int64_t)b * p.delta_sb;
    const T *gz = has_z ? reinterpret_cast<const T *>(p.z) + (int64_t)b * p.z_sb : nullptr;
    const T *gB = varB ? reinterpret_cast<const T *>(p.B) + (int64_t)b * p.B_sb + (int64_t)g * p.B_sg : nullptr;
    const T *gC = varC ? reinterpret_cast<const T *>(p.C) + (int64_t)b * p.C_sb + (int64_t)g * p.C_sg : nullptr;
    T *gout = reinterpret_cast<T *>(p.out) + (int64_t)b * p.out_sb;

    // ---- per-thread constants and state --------------------------------------------------------
    // states live in registers as fp32x2 PAIRS (n, n+1): every FMA-pipe instruction of the inner loop
    // is one zg_f2 pair operation (two scalar fp32 instructions on sm_90a, which has no packed form).
    zg_f2 Al2p[NP], h2[NP];
    float Bc[CONSTBC ? NS : 1], Cc[CONSTBC ? NS : 1];
#pragma unroll
    for (int q = 0; q < NP; ++q) {
        const int n = 2 * q;
        Al2p[q].x = (active && n < N) ? p.A[(int64_t)e * N + n] * ZG_LOG2E : 0.f;
        Al2p[q].y = (active && n + 1 < N) ? p.A[(int64_t)e * N + n + 1] * ZG_LOG2E : 0.f;
        h2[q] = zg_splat2(0.f);
    }
    if (CONSTBC) {
#pragma unroll
        for (int n = 0; n < NS; ++n) {
            Bc[n] = (!varB && active && n < N) ? reinterpret_cast<const float *>(p.B)[(int64_t)e * N + n] : 0.f;
            Cc[n] = (!varC && active && n < N) ? reinterpret_cast<const float *>(p.C)[(int64_t)e * N + n] : 0.f;
        }
    }
    const float Dv = (p.D && active) ? p.D[e] : 0.f;
    const float bias = (p.delta_bias && active) ? p.delta_bias[e] : 0.f;

    const int nstages = (L + TL - 1) / TL;

    // The streaming loads have a fast form (every 16-byte chunk complete and aligned -> bare cp.async,
    // no per-chunk checks) chosen once per CTA, and a generic form for ragged / unaligned tensors.
    bool fast;
    {
        const uintptr_t al = reinterpret_cast<uintptr_t>(p.u) | reinterpret_cast<uintptr_t>(p.delta) | reinterpret_cast<uintptr_t>(p.z) |
                             (varB ? reinterpret_cast<uintptr_t>(p.B) : 0) | (varC ? reinterpret_cast<uintptr_t>(p.C) : 0);
        const int64_t st_or = p.u_sb | p.delta_sb | (has_z ? p.z_sb : 0) | (varB ? (p.B_sb | p.B_sg) : 0) | (varC ? (p.C_sb | p.C_sg) : 0) |
                              (SEQ ? (p.u_sd | p.delta_sd | (has_z ? p.z_sd : 0) | (varB ? p.B_sn : 0) | (varC ? p.C_sn : 0))
                                   : (p.u_sl | p.delta_sl | (has_z ? p.z_sl : 0) | (varB ? p.B_sl : 0) | (varC ? p.C_sl : 0)));
        fast = (al % 16 == 0) && (st_or % VEC == 0) && (e_end - e0 == CH) && (e0 % VEC == 0) && varB && varC &&
               (SEQ ? true : (N == NS));
    }

    // ---- stage loader ---------------------------------------------------------------------------
    auto issue_stage = [&](int s) {
        if (s < nstages) {
            unsigned char *st = smem + (s % NSTAGE) * SM::stage_bytes(NS);
            const int l0 = s * TL;
            const bool full = fast && (l0 + TL <= L);
            if (SEQ) {
                constexpr int CPR = TL * (int)sizeof(T) / 16;      // 16-byte chunks per row
                const int nk = has_z ? 3 : 2;
                for (int it = tid; it < nk * CH * CPR; it += CH) {
                    const int k = it / (CH * CPR), rem = it % (CH * CPR);
                    const int c = rem / CPR, j = rem % CPR;
                    const int ee = e0 + c;
                    const int l = l0 + j * VEC;
                    const T *src = (k == 0) ? gu + (int64_t)ee * p.u_sd + l
                                 : (k == 1) ? gd + (int64_t)ee * p.delta_sd + l
                                            : gz + (int64_t)ee * p.z_sd + l;
                    T *dst = reinterpret_cast<T *>(st + k * SM::ACT_BYTES + c * SM::ACT_ROW_BYTES + j * 16);
                    if (full) {
                        zg_cp_async16(dst, src);
                    } else {
                        if (ee >= e_end) continue;
                        const int nvalid = min(L - l, VEC);
                        if (nvalid > 0) copy_chunk<T>(dst, src, nvalid);
                    }
                }
                // B / C rows: raw[n][TL]
                const int nbc = (varB ? 1 : 0) + (varC ? 1 : 0);
                for (int it = tid; it < nbc * N * CPR; it += CH) {
                    const int w = it / (N * CPR), rem = it % (N * CPR);
                    const int n = rem / CPR, j = rem % CPR;
                    const bool isB = varB && (w == 0);
                    const int l = l0 + j * VEC;
                    const T *src = isB ? gB + (int64_t)n * p.B_sn + l : gC + (int64_t)n * p.C_sn + l;
                    T *dst = reinterpret_cast<T *>(st + 3 * SM::ACT_BYTES + (isB ? 0 : SM::raw_bc_bytes(NS))) + n * TL + j * VEC;
                    if (full) {
                        zg_cp_async16(dst, src);
                    } else {
                        const int nvalid = min(L - l, VEC);
                        if (nvalid > 0) copy_chunk<T>(dst, src, nvalid);
                    }
                }
            } else {
                constexpr int CPR = CH * (int)sizeof(T) / 16;      // chunks per token row
                const int nk = has_z ? 3 : 2;
                for (int it = tid; it < nk * TL * CPR; it += CH) {
                    const int k = it / (TL * CPR), rem = it % (TL * CPR);
                    const int t = rem / CPR, j = rem % CPR;
                    const int l = l0 + t;
                    if (!full && l >= L) continue;
                    const int ee = e0 + j * VEC;
                    const T *src;
                    if (k == 0) src = gu + (int64_t)l * p.u_sl + ee;
                    else if (k == 1) src = gd + (int64_t)l * p.delta_sl + ee;
                    else src = gz + (int64_t)(p.z_rowmap ? p.z_rowmap[l] : l) * p.z_sl + ee;
                    T *dst = reinterpret_cast<T *>(st + k * SM::ACT_BYTES + t * SM::ACT_ROW_BYTES + j * 16);
                    if (full) {
                        zg_cp_async16(dst, src);
                    } else {
                        const int nvalid = min(e_end - ee, VEC);
                        if (nvalid > 0) copy_chunk<T>(dst, src, nvalid);
                    }
                }
                // B / C: raw[t][NS] (state contiguous)
                constexpr int BPR = (NS * (int)sizeof(T) + 15) / 16;
                const int nbc = (varB ? 1 : 0) + (varC ? 1 : 0);
                for (int it = tid; it < nbc * TL * BPR; it += CH) {
                    const int w = it / (TL * BPR), rem = it % (TL * BPR);
                    const int t = rem / BPR, j = rem % BPR;
                    const bool isB = varB && (w == 0);
                    const int l = l0 + t;
                    if (!full && l >= L) continue;
                    const int n0 = j * VEC;
                    const T *src = isB ? gB + (int64_t)l * p.B_sl + n0 : gC + (int64_t)l * p.C_sl + n0;
                    T *dst = reinterpret_cast<T *>(st + 3 * SM::ACT_BYTES + (isB ? 0 : SM::raw_bc_bytes(NS))) + t * NS + n0;
                    if (full) {
                        zg_cp_async16(dst, src);
                    } else {
                        const int nvalid = min(N - n0, VEC);
                        if (nvalid > 0) copy_chunk<T>(dst, src, nvalid);
                    }
                }
            }
        }
        zg_cp_async_commit();
    };

    // ---- SB consecutive recurrence steps (t0 .. t0+SB-1 of the current stage) ------------------------
    // uu/dd/zz: raw inputs of the SB steps; y: results.  The per-step scalars (softplus, delta*u) of the
    // SB steps are independent, so their MUFU latency overlaps; the state update is 4 packed
    // instructions + 2 exp2 per state PAIR and step:
    //     x = dl * A'      a = 2^x      h = a * h + (dl*u) * B      y += C * h
    // The first NPOLY pairs take 2^x from the FMA-pipe polynomial (zg_ex2_poly2), the rest from MUFU.
    auto block = [&](int t0, const float (&uu)[SB], const float (&dd)[SB], const float (&zz)[SB], float (&y)[SB]) {
        zg_f2 dl2[SB], du2[SB], y2[SB];
#pragma unroll
        for (int i = 0; i < SB; ++i) {
            float dl = dd[i] + bias;
            if (softplus) dl = zg_softplus20(dl);
            dl2[i] = zg_splat2(dl);
            du2[i] = zg_splat2(dl * uu[i]);
            y2[i] = zg_pack2(Dv * uu[i], 0.f);
        }
#pragma unroll
        for (int q = 0; q < NP; ++q) {
#pragma unroll
            for (int i = 0; i < SB; ++i) {
                const float2 *bc = reinterpret_cast<const float2 *>(bcf + (t0 + i) * 2 * NS);
                float2 Bv = bc[q], Cv = bc[NP + q];
                if (CONSTBC) {
                    if (!varB) Bv = make_float2(Bc[2 * q], Bc[2 * q + 1]);
                    if (!varC) Cv = make_float2(Cc[2 * q], Cc[2 * q + 1]);
                }
                const zg_f2 x = zg_mul2(dl2[i], Al2p[q]);
                const zg_f2 a = (q < NPOLY) ? zg_ex2_poly2(x) : zg_ex2_mufu2(x);
                h2[q] = zg_fma2(a, h2[q], zg_mul2(du2[i], Bv));
                y2[i] = zg_fma2(Cv, h2[q], y2[i]);
            }
        }
#pragma unroll
        for (int i = 0; i < SB; ++i) {
            float v = y2[i].x + y2[i].y;
            if (has_z) v *= zg_silu(zz[i]);
            y[i] = v;
        }
    };
    auto store_state = [&](float *dst) {
#pragma unroll
        for (int q = 0; q < NP; ++q) {
            if (2 * q < N) dst[2 * q] = h2[q].x;
            if (2 * q + 1 < N) dst[2 * q + 1] = h2[q].y;
        }
    };
    // recompute seeds for the backward pass: the state after every ckpt_every steps (and after the last one)
    const int nck = p.ckpt ? (L + p.ckpt_every - 1) / p.ckpt_every : 0;
    auto ckpt_after = [&](int lend) {      // lend = number of steps done, a multiple of SB or == L
        if (p.ckpt && (lend % p.ckpt_every == 0 || lend == L))
            store_state(p.ckpt + (((int64_t)b * nck + (lend - 1) / p.ckpt_every) * E + e) * N);   // (batch, n_ckpt, dim, dstate)
    };
    // a step beyond the end of the sequence inside a partial block is the identity (delta' = 0 -> a = 1,
    // b = 0), selective_scan_fwd_kernel.cuh:218-222
    const float pad_delta = (softplus ? -1e30f : 0.f) - bias;

    // ---- pipeline -------------------------------------------------------------------------------
#pragma unroll
    for (int s = 0; s < NSTAGE - 1; ++s) issue_stage(s);

    for (int s = 0; s < nstages; ++s) {
        issue_stage(s + NSTAGE - 1);
        zg_cp_async_wait<NSTAGE - 1>();
        __syncthreads();
        unsigned char *st = smem + (s % NSTAGE) * SM::stage_bytes(NS);
        const int l0 = s * TL;
        const int nsteps = min(TL, L - l0);
        const bool full = fast && nsteps == TL;
        // raw B/C (I/O dtype) -> fp32 [t][B0..B(NS-1) C0..C(NS-1)], zero padded
        {
            const T *rawB = reinterpret_cast<const T *>(st + 3 * SM::ACT_BYTES);
            const T *rawC = reinterpret_cast<const T *>(st + 3 * SM::ACT_BYTES + SM::raw_bc_bytes(NS));
            if (!SEQ && full && sizeof(T) == 2 && NS == 16) {
                // one 16-byte chunk (8 states of one step) per thread: 2 (B, C) x 16 steps x 2 halves = 64
                const int w = tid >> 5, t = (tid >> 1) & 15, hf = tid & 1;
                union { uint4 v; T e[8]; } R;
                R.v = *reinterpret_cast<const uint4 *>((w ? rawC : rawB) + t * NS + hf * 8);
                float4 o0, o1;
                o0.x = zg_to_float<T>(R.e[0]); o0.y = zg_to_float<T>(R.e[1]); o0.z = zg_to_float<T>(R.e[2]); o0.w = zg_to_float<T>(R.e[3]);
                o1.x = zg_to_float<T>(R.e[4]); o1.y = zg_to_float<T>(R.e[5]); o1.z = zg_to_float<T>(R.e[6]); o1.w = zg_to_float<T>(R.e[7]);
                float4 *d4 = reinterpret_cast<float4 *>(bcf + t * 2 * NS + w * NS + hf * 8);
                d4[0] = o0; d4[1] = o1;
            } else {
                for (int it = tid; it < 2 * TL * NS; it += CH) {
                    const int w = it / (TL * NS), rem = it % (TL * NS);
                    int t, n;
                    if (SEQ) { n = rem / TL; t = rem % TL; } else { t = rem / NS; n = rem % NS; }
                    float v = 0.f;
                    if (n < N && t < nsteps) {
                        if (w == 0 && varB) v = zg_to_float<T>(SEQ ? rawB[n * TL + t] : rawB[t * NS + n]);
                        if (w == 1 && varC) v = zg_to_float<T>(SEQ ? rawC[n * TL + t] : rawC[t * NS + n]);
                    }
                    bcf[t * 2 * NS + w * NS + n] = v;
                }
            }
        }
        __syncthreads();

        if (active) {
            if (SEQ) {
                // a thread reads 16-byte vectors (VEC steps) along its own smem row; VEC is 4 (fp32) or 8
                const unsigned char *ru = st + 0 * SM::ACT_BYTES + tid * SM::ACT_ROW_BYTES;
                const unsigned char *rd = st + 1 * SM::ACT_BYTES + tid * SM::ACT_ROW_BYTES;
                const unsigned char *rz = st + 2 * SM::ACT_BYTES + tid * SM::ACT_ROW_BYTES;
                T *orow = gout + (int64_t)e * p.out_sd + l0;
#pragma unroll
                for (int tv = 0; tv < TL / VEC; ++tv) {
                    if (tv * VEC >= nsteps) break;
                    union { uint4 v; T e[VEC]; } U, Dl, Z, O;
                    U.v = *reinterpret_cast<const uint4 *>(ru + tv * 16);
                    Dl.v = *reinterpret_cast<const uint4 *>(rd + tv * 16);
                    if (has_z) Z.v = *reinterpret_cast<const uint4 *>(rz + tv * 16);
#pragma unroll
                    for (int sb = 0; sb < VEC / SB; ++sb) {
                        const int t0 = tv * VEC + sb * SB;
                        float uu[SB], dd[SB], zz[SB], y[SB];
                        if (full) {
#pragma unroll
                            for (int i = 0; i < SB; ++i) {
                                uu[i] = zg_to_float<T>(U.e[sb * SB + i]);
                                dd[i] = zg_to_float<T>(Dl.e[sb * SB + i]);
                                zz[i] = has_z ? zg_to_float<T>(Z.e[sb * SB + i]) : 0.f;
                            }
                        } else {
                            if (t0 >= nsteps) continue;
#pragma unroll
                            for (int i = 0; i < SB; ++i) {
                                const bool ok = t0 + i < nsteps;
                                uu[i] = ok ? zg_to_float<T>(U.e[sb * SB + i]) : 0.f;
                                dd[i] = ok ? zg_to_float<T>(Dl.e[sb * SB + i]) : pad_delta;
                                zz[i] = (ok && has_z) ? zg_to_float<T>(Z.e[sb * SB + i]) : 0.f;
                            }
                        }
                        block(t0, uu, dd, zz, y);
                        ckpt_after(min(l0 + t0 + SB, L));
#pragma unroll
                        for (int i = 0; i < SB; ++i) O.e[sb * SB + i] = zg_from_float<T>(y[i]);
                    }
                    T *dst = orow + tv * VEC;
                    if (full || (tv * VEC + VEC <= nsteps && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0))) {
                        *reinterpret_cast<uint4 *>(dst) = O.v;
                    } else {
#pragma unroll
                        for (int i = 0; i < VEC; ++i)
                            if (tv * VEC + i < nsteps) dst[i] = O.e[i];
                    }
                }
            } else {
                const T *su = reinterpret_cast<const T *>(st + 0 * SM::ACT_BYTES) + tid;
                const T *sd = reinterpret_cast<const T *>(st + 1 * SM::ACT_BYTES) + tid;
                const T *sz = reinterpret_cast<const T *>(st + 2 * SM::ACT_BYTES) + tid;
                T *ocol = gout + (int64_t)l0 * p.out_sl + e;
                if (nsteps == TL) {
#pragma unroll 1
                    for (int t0 = 0; t0 < TL; t0 += SB) {
                        float uu[SB], dd[SB], zz[SB], y[SB];
#pragma unroll
                        for (int i = 0; i < SB; ++i) {
                            uu[i] = zg_to_float<T>(su[(t0 + i) * CH]);
                            dd[i] = zg_to_float<T>(sd[(t0 + i) * CH]);
                            zz[i] = has_z ? zg_to_float<T>(sz[(t0 + i) * CH]) : 0.f;
                        }
                        block(t0, uu, dd, zz, y);
                        ckpt_after(min(l0 + t0 + SB, L));
#pragma unroll
                        for (int i = 0; i < SB; ++i) ocol[(int64_t)(t0 + i) * p.out_sl] = zg_from_float<T>(y[i]);
                    }
                } else {
#pragma unroll 1
                    for (int t0 = 0; t0 < nsteps; t0 += SB) {
                        float uu[SB], dd[SB], zz[SB], y[SB];
#pragma unroll
                        for (int i = 0; i < SB; ++i) {
                            const bool ok = t0 + i < nsteps;
                            uu[i] = ok ? zg_to_float<T>(su[(t0 + i) * CH]) : 0.f;
                            dd[i] = ok ? zg_to_float<T>(sd[(t0 + i) * CH]) : pad_delta;
                            zz[i] = (ok && has_z) ? zg_to_float<T>(sz[(t0 + i) * CH]) : 0.f;
                        }
                        block(t0, uu, dd, zz, y);
                        ckpt_after(min(l0 + t0 + SB, L));
#pragma unroll
                        for (int i = 0; i < SB; ++i)
                            if (t0 + i < nsteps) ocol[(int64_t)(t0 + i) * p.out_sl] = zg_from_float<T>(y[i]);
                    }
                }
            }
        }
        __syncthreads();   // stage buffer and bcf are recycled by the next iteration
    }

    if (active && p.last_state) store_state(p.last_state + ((int64_t)b * E + e) * N);
}

template <typename T, int NS, bool SEQ, bool CONSTBC, int NPOLY = 0>
int launch_scan_fwd(const zg_scan_params &p, cudaStream_t stream) {
    using SM = ScanSmem<T, SEQ>;
    const int per_group = p.dim / p.ngroups;
    const int tiles = p.ngroups * ((per_group + SCAN_CH - 1) / SCAN_CH);
    const int smem = SM::total_bytes(NS);
    auto kern = scan_fwd_kernel<T, NS, SEQ, CONSTBC, NPOLY>;
    static bool attr_set = false;   // per instantiation
    if (!attr_set) {
        cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (err != cudaSuccess) return zg_set_error("scan_fwd: cudaFuncSetAttribute(%d B smem): %s", smem, cudaGetErrorString(err));
        // all of the SM's unified L1/shared array as shared memory: 9-10 CTAs x (stage ring + 1 KB) must fit
        cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        attr_set = true;
    }
    const long long nblk = (long long)tiles * p.batch;
    if (nblk > 0x7fffffffLL) return zg_set_error("scan_fwd: grid too large (%lld CTAs)", nblk);
    if (nblk == 0) return 0;
    kern<<<(unsigned)nblk, SCAN_CH, smem, stream>>>(p);
    zg_count_launch();
    zg_note_scan_kernel("zg::scan_fwd_kernel (generic: one thread per channel)");
    return zg_check_launch("scan_fwd");
}

// How many state pairs use the polynomial exp2 (tuning knob; default carried over from measurements on another GPU; not re-tuned on H100
// in DESIGN.md).  ZG_SCAN_NPOLY in the environment overrides it (read once).
inline int scan_npoly_setting() {
    static int v = -1;
    if (v < 0) {
        const char *e = getenv("ZG_SCAN_NPOLY");
        v = e ? atoi(e) : ZG_SCAN_NPOLY_DEFAULT;
        if (v != 0 && v != 2 && v != 3 && v != 4) v = ZG_SCAN_NPOLY_DEFAULT;
    }
    return v;
}

// one translation unit per I/O dtype (parallel compilation)
template <typename T, int NS, bool SEQ> int launch_scan_fwd_npoly(const zg_scan_params &p, cudaStream_t stream) {
    if (NS == 16) {
        switch (scan_npoly_setting()) {
            case 2: return launch_scan_fwd<T, NS, SEQ, false, (NS == 16 ? 2 : 0)>(p, stream);
            case 3: return launch_scan_fwd<T, NS, SEQ, false, (NS == 16 ? 3 : 0)>(p, stream);
            case 4: return launch_scan_fwd<T, NS, SEQ, false, (NS == 16 ? 4 : 0)>(p, stream);
            default: break;
        }
    }
    return launch_scan_fwd<T, NS, SEQ, false, 0>(p, stream);
}

// Pure part of scan_auto_choice (scan_fwd_tma.cuh; exported as zg_scan_kernel_choice so that the rule is testable without a GPU):
// U 16-channel units, S SMs, ckpt = the training forward.  mode 0: CTA-wide kernel, 3: 32-channel warps, 5: mixed CTAs of nd wide +
// ns narrow warps.
struct ScanChoice { int mode, nd, ns; };
inline ScanChoice scan_choice_for(long long U, long long S, bool ckpt) {
    if (ckpt || S <= 0) return {0, 0, 0};
    if (U < 16 * S) return {0, 0, 0};      // under four units per sub-partition nothing saturates the pipe: the narrow warps' shorter steps win (batch 16: 0.211 vs 0.229 ms)
    if (U > 36 * S) return {3, 0, 0};
    const long long base = ((U + 3) / 4 + S - 1) / S;
    const long long wide = 2 * ((((U + 1) / 2 + S - 1) / S + 3) / 4);
    if (wide <= base) return {3, 0, 0};
    const long long per_cta = (((U + S - 1) / S + 1) / 2 + 1) & ~1LL;      // units per CTA, two CTAs per SM, even
    for (int nd = 8; nd >= 4; nd -= 4) {                                   // wide warps in multiples of 4 (one per sub-partition), at most 10 warps
        const long long ns = per_cta - 2 * nd;
        if (ns >= 0 && (ns & 1) == 0 && nd + ns <= 10 && per_cta / 2 <= base) return {5, nd, (int)ns};
    }
    return {0, 0, 0};
}

template <typename T> int try_launch_scan_fwd_tpc2(const zg_scan_params &p, cudaStream_t stream);   // scan_fwd_tpc2.cuh
template <typename T> int try_launch_scan_fwd_tma(const zg_scan_params &p, cudaStream_t stream);    // scan_fwd_tma.cuh

template <typename T> int dispatch_scan_fwd(const zg_scan_params &p, bool seq, bool constbc, cudaStream_t stream) {
    const int N = p.dstate;
    if constexpr (sizeof(T) == 2) {
        if (!seq && !constbc) {     // hot-path specialisations, when the call fits them: round 2 (bulk-async pipeline), round 1
            int rc = try_launch_scan_fwd_tma<T>(p, stream);
            if (rc >= 0) return rc;
            if (p.dt_w || p.z_batch_inner > 0 || (p.flags & (ZG_SCAN_OUT_REVERSE | ZG_SCAN_OUT_ACCUMULATE))) goto unsupported;   // only that kernel implements them
            rc = try_launch_scan_fwd_tpc2<T>(p, stream);
            if (rc >= 0) return rc;
        }
    }
unsupported:
    if (p.dt_w) return zg_set_error("selective_scan_fwd: the fused dt_proj prologue needs 16-bit dim-contiguous activations with input-dependent B/C");
    if (p.z_batch_inner > 0) return zg_set_error("selective_scan_fwd: z_batch_inner is implemented by the hot-path kernel only (16-bit dim-contiguous, dstate 16, seqlen %% 8 == 0, dim %% 64 == 0, z_rowmap given)");
    if (p.flags & (ZG_SCAN_OUT_REVERSE | ZG_SCAN_OUT_ACCUMULATE))
        return zg_set_error("selective_scan_fwd: OUT_REVERSE / OUT_ACCUMULATE are implemented by the hot-path kernel only (16-bit dim-contiguous, dstate 16, seqlen %% 8 == 0, dim %% 64 == 0)");
#define ZG_SCAN_CASE(NSV)                                                                   \
    if (N <= NSV) {                                                                         \
        if (seq) return launch_scan_fwd_npoly<T, NSV, true>(p, stream);                     \
        return launch_scan_fwd_npoly<T, NSV, false>(p, stream);                             \
    }
    if (constbc) {
        if (N <= 8) return seq ? launch_scan_fwd<T, 8, true, true>(p, stream) : launch_scan_fwd<T, 8, false, true>(p, stream);
        if (N <= 16) return seq ? launch_scan_fwd<T, 16, true, true>(p, stream) : launch_scan_fwd<T, 16, false, true>(p, stream);
        return zg_set_error("selective_scan_fwd: constant (non input-dependent) B/C supports dstate <= 16, got %d", N);
    }
    ZG_SCAN_CASE(8)
    ZG_SCAN_CASE(16)
    ZG_SCAN_CASE(32)
    ZG_SCAN_CASE(64)
#undef ZG_SCAN_CASE
    return zg_set_error("selective_scan_fwd: dstate %d > 64 not supported", N);
}

int scan_fwd_f32(const zg_scan_params &p, bool seq, bool constbc, cudaStream_t s);
int scan_fwd_f16(const zg_scan_params &p, bool seq, bool constbc, cudaStream_t s);
int scan_fwd_bf16(const zg_scan_params &p, bool seq, bool constbc, cudaStream_t s);

}  // namespace zg
