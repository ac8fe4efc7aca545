// Selective-scan backward, dstate == 16 specialisation for sm_90a: FOUR threads per channel, four
// states each ("quad" = lanes 4j..4j+3 of a warp), 64 channels x one batch row per 256-thread CTA.
// Same math as the generic kernel in scan_bwd.cu (reference: selective_scan_bwd_kernel.cuh:186-213,
// 252-296,439-452); what changes is the mapping, chosen for occupancy and memory behaviour:
//
//   * parked states (h_{l-1} of the 8 steps of a chunk, recomputed from the forward's checkpoint)
//     cost 64 B per (channel, step) whatever the thread mapping -- with 4 threads per channel that is
//     128 B per THREAD, so 4 CTAs = 32 warps fit an SM (the one-thread-per-channel kernel: 6 warps);
//     one LDS.128 / STS.128 per thread-step, conflict free ([step][channel][quad] float4);
//   * every global access goes through a per-chunk cooperative prologue / epilogue, so it is coalesced
//     for BOTH layouts the ABI allows (channel-first (b, d, l) as the reference's autograd passes,
//     token-major (b l, d) as the engine uses) and each softplus / sigmoid is evaluated ONCE per
//     (channel, step), not once per thread of the quad;
//   * STAGED variant (aligned shapes, i.e. every real model): the raw inputs of the NEXT chunk are fetched
//     with 16-byte cp.async into a staging buffer while the current chunk is recomputed and swept, so no
//     warp waits on a global load (ncu round 1, unstaged: a third of the stall samples sat on the first
//     use of the prologue's loads); outputs leave as 4-byte pairs;
//   * dB / dC (sums over the channels that share a group): 7-shuffle transpose-reduce over the 8
//     channels of a warp, cross-warp sum through shared memory, then one fp32 atomic per
//     (CTA, state, step) with 8 consecutive steps per 32-byte sector;
//   * zg_f2 pair math on state pairs, as in the forward;
//   * z_rowmap (the forward's fused permutation of the gate) redirects the z reads and the dz writes.
#pragma once
#include "zg_common.cuh"

namespace zg {

constexpr int Q4_CH = 64;          // channels per CTA
constexpr int Q4_THREADS = 256;
constexpr int Q4_TS = 8;           // steps per chunk == ckpt_every of the forward
constexpr int Q4_RED_LD = Q4_TS + 1;

template <typename T, bool STAGED> struct Q4Smem {
    static constexpr int HS = Q4_TS * Q4_CH * 4 * 16;              // float4 [TS][CH][4]
    static constexpr int SC = Q4_TS * Q4_CH * 16;                  // float4 [TS][CH]  (delta', u, dy, gz) -> (du, ddelta, dz, -)
    static constexpr int BC = Q4_TS * 32 * 4;                      // float  [TS][B0..15 C0..15]
    static constexpr int RED = 8 * 32 * Q4_RED_LD * 4;             // float  [warp][slot][TS+1]
    static constexpr int ACT = Q4_TS * Q4_CH * (int)sizeof(T);     // one staged activation tile (raw)
    static constexpr int STG = STAGED ? 4 * ACT + 2 * Q4_TS * 16 * (int)sizeof(T) : 0;
    static constexpr int TOTAL = HS + SC + BC + RED + STG;
};

template <typename T> __device__ __forceinline__ float2 q4_ld_pair(const unsigned char *p);
template <> __device__ __forceinline__ float2 q4_ld_pair<float>(const unsigned char *p) { return *reinterpret_cast<const float2 *>(p); }
template <> __device__ __forceinline__ float2 q4_ld_pair<__half>(const unsigned char *p) { return __half22float2(*reinterpret_cast<const __half2 *>(p)); }
template <> __device__ __forceinline__ float2 q4_ld_pair<__nv_bfloat16>(const unsigned char *p) {
    const unsigned r = *reinterpret_cast<const unsigned *>(p);
    return make_float2(__uint_as_float(r << 16), __uint_as_float(r & 0xffff0000u));
}
template <typename T> __device__ __forceinline__ void q4_st_pair(T *p, float a, float b);
template <> __device__ __forceinline__ void q4_st_pair<float>(float *p, float a, float b) { *reinterpret_cast<float2 *>(p) = make_float2(a, b); }
template <> __device__ __forceinline__ void q4_st_pair<__half>(__half *p, float a, float b) { *reinterpret_cast<__half2 *>(p) = __floats2half2_rn(a, b); }
template <> __device__ __forceinline__ void q4_st_pair<__nv_bfloat16>(__nv_bfloat16 *p, float a, float b) {
    *reinterpret_cast<__nv_bfloat162 *>(p) = __floats2bfloat162_rn(a, b);
}

// DET: the gradient pointers of q address partial rows instead of the outputs (zg_selective_scan_bwd_det): dB / dC one
// row per channel tile within the group, (tiles_per_group, batch, groups, 16, seqlen); dA / dD / d(delta_bias) one row per
// batch row, (batch, dim, 16) / (batch, dim); plain stores where the atomic path adds.
template <typename T, bool STAGED, bool DET>
__global__ void __launch_bounds__(Q4_THREADS, 4) scan_bwd_q4_kernel(const zg_scan_bwd_params q) {
    const zg_scan_params &p = q.fwd;
    constexpr int TS = Q4_TS, CH = Q4_CH;
    using SM = Q4Smem<T, STAGED>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float4 *hs = reinterpret_cast<float4 *>(smem_raw);
    float4 *sc = reinterpret_cast<float4 *>(smem_raw + SM::HS);
    float *bcf = reinterpret_cast<float *>(smem_raw + SM::HS + SM::SC);
    float *red = bcf + TS * 32;
    unsigned char *stg = smem_raw + SM::HS + SM::SC + SM::BC + SM::RED;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int c = tid >> 2, qd = tid & 3;                   // channel within the CTA, quarter of the state vector
    const int E = p.dim, L = p.seqlen;
    const int per_group = E / p.ngroups;
    const int tiles_per_group = (per_group + CH - 1) / CH;
    const int tiles = tiles_per_group * p.ngroups;
    const int b = blockIdx.x / tiles;
    const int tile = blockIdx.x % tiles;
    const int g = tile / tiles_per_group;
    const int e0 = g * per_group + (tile % tiles_per_group) * CH;
    const int e_end = min(e0 + CH, (g + 1) * per_group);
    const bool active = e0 + c < e_end;
    const int e = active ? e0 + c : e0;
    const bool has_z = p.z != nullptr;
    const bool softplus = (p.flags & ZG_SCAN_DELTA_SOFTPLUS) != 0;

    // ---- cooperative (prologue / epilogue) item mapping: 64 channels x 8 steps = 2 items per thread --------
    // token-major tensors: consecutive threads -> consecutive channels; channel-first: consecutive steps.
    // STAGED: the two items are neighbours (a channel pair / a step pair) so that they travel as one 4-byte word.
    const bool tok = (p.u_sd == 1);
    int ic[2], it[2];
    if (STAGED) {
        if (tok) { it[0] = it[1] = tid >> 5; ic[0] = 2 * (tid & 31); ic[1] = ic[0] + 1; }
        else { ic[0] = ic[1] = tid >> 2; it[0] = 2 * (tid & 3); it[1] = it[0] + 1; }
    } else {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int i = tid + j * Q4_THREADS;
            ic[j] = tok ? (i & (CH - 1)) : (i >> 3);
            it[j] = tok ? (i >> 6) : (i & 7);
        }
    }
    float ibias[2];
    bool ich_ok[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        ich_ok[j] = e0 + ic[j] < e_end;
        ibias[j] = (p.delta_bias && ich_ok[j]) ? p.delta_bias[e0 + ic[j]] : 0.f;
    }
    const T *gu = reinterpret_cast<const T *>(p.u) + (int64_t)b * p.u_sb + (int64_t)e0 * p.u_sd;
    const T *gd = reinterpret_cast<const T *>(p.delta) + (int64_t)b * p.delta_sb + (int64_t)e0 * p.delta_sd;
    const T *gz = has_z ? reinterpret_cast<const T *>(p.z) + (int64_t)b * p.z_sb + (int64_t)e0 * p.z_sd : nullptr;
    const T *gdo = reinterpret_cast<const T *>(q.dout) + (int64_t)b * q.dout_sb + (int64_t)e0 * q.dout_sd;
    const T *gB = reinterpret_cast<const T *>(p.B) + (int64_t)b * p.B_sb + (int64_t)g * p.B_sg;
    const T *gC = reinterpret_cast<const T *>(p.C) + (int64_t)b * p.C_sb + (int64_t)g * p.C_sg;
    T *gdu = reinterpret_cast<T *>(q.du) + (int64_t)b * q.du_sb + (int64_t)e0 * q.du_sd;
    T *gdd = reinterpret_cast<T *>(q.ddelta) + (int64_t)b * q.ddelta_sb + (int64_t)e0 * q.ddelta_sd;
    T *gdz = has_z ? reinterpret_cast<T *>(q.dz) + (int64_t)b * q.dz_sb + (int64_t)e0 * q.dz_sd : nullptr;
    const int64_t det_row = DET ? (int64_t)(tile % tiles_per_group) * p.batch * p.ngroups * 16 * L : 0;
    float *gdB = q.dB + det_row + ((int64_t)b * p.ngroups + g) * (int64_t)16 * L;      // (batch, groups, dstate, seqlen)
    float *gdC = q.dC + det_row + ((int64_t)b * p.ngroups + g) * (int64_t)16 * L;
    const int nck = (L + TS - 1) / TS;
    const float4 *ck = reinterpret_cast<const float4 *>(p.ckpt + ((int64_t)b * nck * E + e) * (int64_t)16) + qd;   // (batch, n_ckpt, dim, 16)
    // B / C: 2 x 8 steps x 16 states = 256 values, one per thread
    const int bw = tid >> 7, brem = tid & 127;
    const bool bc_tok = (bw ? p.C_sn : p.B_sn) == 1;
    const int bn = bc_tok ? (brem & 15) : (brem >> 3), bt = bc_tok ? (brem >> 4) : (brem & 7);
    const T *gbc = bw ? gC + (int64_t)bn * p.C_sn : gB + (int64_t)bn * p.B_sn;
    const int64_t bc_sl = bw ? p.C_sl : p.B_sl;

    // ---- STAGED: cp.async of one chunk's raw inputs (in-batch offsets fit 32 bits, checked on the host) --------
    // activation tile layout = source layout: token-major [t][c], channel-first [c][t]; B | C raw likewise
    auto issue_stage = [&](int k) {
        constexpr int EPC = 16 / (int)sizeof(T);                     // elements per 16-byte chunk
        constexpr int NPT = TS * CH / EPC;                           // chunks per activation tile
        const int l0 = k * TS;
        for (int i = tid; i < 4 * NPT; i += Q4_THREADS) {
            const int tensor = i / NPT, idx = i % NPT;
            if (tensor == 3 && !has_z) break;
            const T *base = tensor == 0 ? gd : tensor == 1 ? gu : tensor == 2 ? gdo : gz;
            const int sl = (int)(tensor == 0 ? p.delta_sl : tensor == 1 ? p.u_sl : tensor == 2 ? q.dout_sl : p.z_sl);
            const int sd = (int)(tensor == 0 ? p.delta_sd : tensor == 1 ? p.u_sd : tensor == 2 ? q.dout_sd : p.z_sd);
            int off;
            if (tok) {
                const int t = idx / (CH / EPC), j = idx % (CH / EPC);
                const int l = l0 + t;
                off = ((tensor == 3 && p.z_rowmap) ? p.z_rowmap[l] : l) * sl + j * EPC;
            } else {
                const int cc = idx / (TS / EPC), j = idx % (TS / EPC);
                off = cc * sd + l0 + j * EPC;
            }
            zg_cp_async16(stg + tensor * SM::ACT + idx * 16, base + off);
        }
        constexpr int NBC = 2 * TS * 16 / EPC;                       // 32 (16-bit) or 64 (fp32) chunks for B | C
        if (tid < NBC) {
            const int w = tid / (NBC / 2), idx = tid % (NBC / 2);
            const T *base = w ? gC : gB;
            const int sn = (int)(w ? p.C_sn : p.B_sn), sl = (int)(w ? p.C_sl : p.B_sl);
            int off;
            if (sn == 1) { const int t = idx / (16 / EPC), j = idx % (16 / EPC); off = (l0 + t) * sl + j * EPC; }
            else { const int n = idx / (TS / EPC), j = idx % (TS / EPC); off = n * sn + l0 + j * EPC; }
            zg_cp_async16(stg + 4 * SM::ACT + (w * (NBC / 2) + idx) * 16, base + off);
        }
        zg_cp_async_commit();
    };

    // ---- per-thread state: 4 states as two packed pairs --------------------------------------------------
    zg_f2 A2[2], dA[2], carry[2];
    {
        const float4 a4 = *reinterpret_cast<const float4 *>(p.A + (int64_t)e * 16 + 4 * qd);
        A2[0] = make_float2(a4.x * ZG_LOG2E, a4.y * ZG_LOG2E);
        A2[1] = make_float2(a4.z * ZG_LOG2E, a4.w * ZG_LOG2E);
    }
    dA[0] = dA[1] = carry[0] = carry[1] = zg_splat2(0.f);
    const float Dv = p.D ? p.D[e] : 0.f;
    float dD_acc = 0.f, dbias_acc = 0.f;                    // meaningful in the qd == 0 thread

    if (STAGED) issue_stage(nck - 1);

    for (int k = nck - 1; k >= 0; --k) {
        const int l0 = k * TS;
        // ---- prologue: inputs -> per-(step, channel) scalars in shared memory ------------------------------
        if (STAGED) {
            zg_cp_async_wait<0>();
            __syncthreads();            // staged bytes visible; everybody is done with the previous chunk's sc / red
            const int po = (tok ? it[0] * CH + ic[0] : ic[0] * TS + it[0]) * (int)sizeof(T);
            const float2 dd2 = q4_ld_pair<T>(stg + po), uu2 = q4_ld_pair<T>(stg + SM::ACT + po), do2 = q4_ld_pair<T>(stg + 2 * SM::ACT + po);
            float2 zz2 = make_float2(0.f, 0.f);
            if (has_z) zz2 = q4_ld_pair<T>(stg + 3 * SM::ACT + po);
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                float d = (j ? dd2.y : dd2.x) + ibias[j];
                if (softplus) d = zg_softplus20(d);
                const float dout = j ? do2.y : do2.x;
                float4 s = make_float4(d, j ? uu2.y : uu2.x, dout, 0.f);
                if (has_z) {
                    const float zz = j ? zz2.y : zz2.x;
                    const float sg = zg_sigmoid(zz);
                    s.z = dout * zz * sg;
                    s.w = dout * sg * (1.f + zz * (1.f - sg));
                }
                sc[it[j] * CH + ic[j]] = s;
            }
            bcf[bt * 32 + bw * 16 + bn] = zg_to_float<T>(reinterpret_cast<const T *>(stg + 4 * SM::ACT)[tid]);
        } else {
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const int l = l0 + it[j];
                float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
                if (ich_ok[j] && l < L) {
                    float d = zg_to_float<T>(gd[(int64_t)ic[j] * p.delta_sd + (int64_t)l * p.delta_sl]) + ibias[j];
                    if (softplus) d = zg_softplus20(d);
                    const float dout = zg_to_float<T>(gdo[(int64_t)ic[j] * q.dout_sd + (int64_t)l * q.dout_sl]);
                    s.x = d;
                    s.y = zg_to_float<T>(gu[(int64_t)ic[j] * p.u_sd + (int64_t)l * p.u_sl]);
                    s.z = dout;
                    if (has_z) {
                        const int64_t lz = p.z_rowmap ? p.z_rowmap[l] : l;       // z is read (and dz written) in token order
                        const float zz = zg_to_float<T>(gz[(int64_t)ic[j] * p.z_sd + lz * p.z_sl]);
                        const float sg = zg_sigmoid(zz);
                        s.z = dout * zz * sg;
                        s.w = dout * sg * (1.f + zz * (1.f - sg));
                    }
                }
                sc[it[j] * CH + ic[j]] = s;
            }
            const int l = l0 + bt;
            bcf[bt * 32 + bw * 16 + bn] = (l < L) ? zg_to_float<T>(gbc[(int64_t)l * bc_sl]) : 0.f;
        }
        __syncthreads();
        if (STAGED && k > 0) issue_stage(k - 1);          // in flight during the recompute and the sweep below

        // ---- forward recompute from the checkpoint before the chunk, parking h_{l-1} -----------------------
        zg_f2 h[2];
        if (k > 0) {
            const float4 h4 = ck[(int64_t)(k - 1) * E * 4];
            h[0] = make_float2(h4.x, h4.y); h[1] = make_float2(h4.z, h4.w);
        } else {
            h[0] = h[1] = zg_splat2(0.f);
        }
        {
            const float4 *scp = sc + c;
            const float *bcp = bcf + 4 * qd;
            float4 *hsp = hs + c * 4 + qd;
#pragma unroll 1
            for (int t = 0; t < TS; ++t, scp += CH, bcp += 32, hsp += CH * 4) {
                const float4 s = *scp;
                const float4 B4 = *reinterpret_cast<const float4 *>(bcp);
                *hsp = make_float4(h[0].x, h[0].y, h[1].x, h[1].y);
                const zg_f2 d2 = zg_splat2(s.x), ddu2 = zg_splat2(s.x * s.y);
                h[0] = zg_fma2(zg_ex2_mufu2(zg_mul2(d2, A2[0])), h[0], zg_mul2(ddu2, make_float2(B4.x, B4.y)));
                h[1] = zg_fma2(zg_ex2_mufu2(zg_mul2(d2, A2[1])), h[1], zg_mul2(ddu2, make_float2(B4.z, B4.w)));
            }
        }

        // ---- reverse sweep -------------------------------------------------------------------------------------
        {
            float4 *scp = sc + (TS - 1) * CH + c;
            const float *bcp = bcf + (TS - 1) * 32 + 4 * qd;
            const float4 *hsp = hs + ((TS - 1) * CH + c) * 4 + qd;
            const int vi = lane >> 2;
            float *redp = red + (warp * 32 + ((vi & 4) << 2) + 4 * qd + (vi & 3)) * Q4_RED_LD + (TS - 1);   // slot = [dB0..15 | dC0..15]
#pragma unroll 1     // (full unrolling spills at the 64-register budget of 4 CTAs / SM)
            for (int t = TS - 1; t >= 0; --t, scp -= CH, bcp -= 32, hsp -= CH * 4, --redp) {
                const float4 s = *scp;                                // delta', u, dy, gz
                const float4 B4 = *reinterpret_cast<const float4 *>(bcp);
                const float4 C4 = *reinterpret_cast<const float4 *>(bcp + 16);
                const float4 hp4 = *hsp;
                const zg_f2 Bp[2] = {make_float2(B4.x, B4.y), make_float2(B4.z, B4.w)};
                const zg_f2 Cp[2] = {make_float2(C4.x, C4.y), make_float2(C4.z, C4.w)};
                const zg_f2 hp[2] = {make_float2(hp4.x, hp4.y), make_float2(hp4.z, hp4.w)};
                const zg_f2 d2 = zg_splat2(s.x), ddu2 = zg_splat2(s.x * s.y), dy2 = zg_splat2(s.z);
                zg_f2 y2 = zg_splat2(0.f), s1 = zg_splat2(0.f), s2 = zg_splat2(0.f);
                float v[8];                                           // dB[4qd..4qd+3] | dC[4qd..4qd+3] of this channel
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const zg_f2 a = zg_ex2_mufu2(zg_mul2(d2, A2[i]));
                    const zg_f2 hl = zg_fma2(a, hp[i], zg_mul2(ddu2, Bp[i]));
                    y2 = zg_fma2(Cp[i], hl, y2);
                    const zg_f2 dh = zg_fma2(dy2, Cp[i], carry[i]);   // dh_l = dy_l C_l + a_{l+1} dh_{l+1}
                    carry[i] = zg_mul2(a, dh);
                    const zg_f2 t1 = zg_mul2(carry[i], hp[i]);        // dh_l a_l h_{l-1}
                    s1 = zg_fma2(dh, Bp[i], s1);
                    s2 = zg_fma2(t1, A2[i], s2);
                    dA[i] = zg_fma2(t1, d2, dA[i]);
                    const zg_f2 vb = zg_mul2(dh, ddu2), vc = zg_mul2(dy2, hl);
                    v[2 * i] = vb.x; v[2 * i + 1] = vb.y; v[4 + 2 * i] = vc.x; v[4 + 2 * i + 1] = vc.y;
                }
                float yq = y2.x + y2.y, s1q = s1.x + s1.y, s2q = s2.x + s2.y;
#pragma unroll
                for (int o = 1; o <= 2; o <<= 1) {
                    yq += __shfl_xor_sync(0xffffffffu, yq, o);
                    s1q += __shfl_xor_sync(0xffffffffu, s1q, o);
                    s2q += __shfl_xor_sync(0xffffffffu, s2q, o);
                }
                __syncwarp();        // the quad has read *scp (compute-sanitizer racecheck: WAR hazard without it)
                if (qd == 0) {
                    const float du_ = fmaf(s.x, s1q, s.z * Dv);
                    float dd = fmaf(s2q, ZG_LN2, s.y * s1q);
                    if (softplus) dd *= zg_softplus_grad(s.x);   // sigmoid(delta~) = 1 - exp(-softplus(delta~))
                    dD_acc = fmaf(s.z, s.y, dD_acc);
                    dbias_acc += dd;
                    *scp = make_float4(du_, dd, s.w * fmaf(Dv, s.y, yq), 0.f);   // the slot now carries the outputs
                }
                // transpose-reduce the 8 values over the 8 channels of the warp (lane bits 4, 3, 2): afterwards the
                // lane of channel j holds the total of value j
#pragma unroll
                for (int half = 4; half >= 1; half >>= 1) {
                    const bool up = (lane & (half << 2)) != 0;
#pragma unroll
                    for (int j = 0; j < half; ++j) {
                        const float send = up ? v[j] : v[j + half];
                        const float keep = up ? v[j + half] : v[j];
                        v[j] = keep + __shfl_xor_sync(0xffffffffu, send, half << 2);
                    }
                }
                *redp = v[0];
            }
        }
        __syncthreads();

        // ---- epilogue: coalesced stores + one atomic per (state, step) ----------------------------------------
        if (STAGED) {
            const float4 o0 = sc[it[0] * CH + ic[0]], o1 = sc[it[1] * CH + ic[1]];
            const int l = l0 + it[0];
            q4_st_pair<T>(gdu + ic[0] * (int)q.du_sd + l * (int)q.du_sl, o0.x, o1.x);
            q4_st_pair<T>(gdd + ic[0] * (int)q.ddelta_sd + l * (int)q.ddelta_sl, o0.y, o1.y);
            if (has_z) q4_st_pair<T>(gdz + ic[0] * (int)q.dz_sd + (p.z_rowmap ? p.z_rowmap[l] : l) * (int)q.dz_sl, o0.z, o1.z);
        } else {
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const int l = l0 + it[j];
                if (ich_ok[j] && l < L) {
                    const float4 o = sc[it[j] * CH + ic[j]];
                    gdu[(int64_t)ic[j] * q.du_sd + (int64_t)l * q.du_sl] = zg_from_float<T>(o.x);
                    gdd[(int64_t)ic[j] * q.ddelta_sd + (int64_t)l * q.ddelta_sl] = zg_from_float<T>(o.y);
                    if (has_z) {
                        const int64_t lz = p.z_rowmap ? p.z_rowmap[l] : l;
                        gdz[(int64_t)ic[j] * q.dz_sd + lz * q.dz_sl] = zg_from_float<T>(o.z);
                    }
                }
            }
        }
        {
            const int slot = tid >> 3, t = tid & 7, l = l0 + t;
            float acc = 0.f;
#pragma unroll
            for (int w = 0; w < 8; ++w) acc += red[(w * 32 + slot) * Q4_RED_LD + t];
            if (l < L) {
                float *dst = (slot < 16 ? gdB : gdC) + (int64_t)(slot & 15) * L + l;
                if constexpr (DET) *dst = acc;
                else atomicAdd(dst, acc);
            }
        }
        if (!STAGED) __syncthreads();      // (STAGED: the barrier at the top of the next iteration does this job)
    }

    if (DET && active) {
        const int64_t be = (int64_t)b * E + e;
        *reinterpret_cast<float4 *>(q.dA + be * 16 + 4 * qd) = make_float4(dA[0].x, dA[0].y, dA[1].x, dA[1].y);
        if (qd == 0) {
            if (q.dD) q.dD[be] = dD_acc;
            if (q.ddelta_bias) q.ddelta_bias[be] = dbias_acc;
        }
    } else if (active) {
        float *dAe = q.dA + (int64_t)e * 16 + 4 * qd;
        atomicAdd(dAe + 0, dA[0].x); atomicAdd(dAe + 1, dA[0].y);
        atomicAdd(dAe + 2, dA[1].x); atomicAdd(dAe + 3, dA[1].y);
        if (qd == 0) {
            if (q.dD) atomicAdd(q.dD + e, dD_acc);
            if (q.ddelta_bias) atomicAdd(q.ddelta_bias + e, dbias_acc);
        }
    }
}

// whether a call runs the dstate == 16 kernel (else the generic one in scan_bwd.cu); host arithmetic only
static inline bool scan_bwd_q4_fits(const zg_scan_bwd_params &q) {
    static int enabled = -1;
    if (enabled < 0) { const char *e = getenv("ZG_SCAN_BWD_Q4"); enabled = e ? atoi(e) : 1; }
    const zg_scan_params &p = q.fwd;
    if (!enabled || p.dstate != 16 || p.ckpt_every != Q4_TS) return false;
    if (!(p.flags & ZG_SCAN_VARIABLE_B) || !(p.flags & ZG_SCAN_VARIABLE_C)) return false;      // constant B / C: the generic kernel
    if ((reinterpret_cast<uintptr_t>(p.A) | reinterpret_cast<uintptr_t>(p.ckpt)) % 16 != 0) return false;
    const int per_group = p.dim / p.ngroups;
    const long long nblk = (long long)p.ngroups * ((per_group + Q4_CH - 1) / Q4_CH) * p.batch;
    return nblk <= 0x7fffffffLL;
}

// returns -1 when the call does not fit this specialisation
template <typename T, bool DET = false> int try_launch_scan_bwd_q4(const zg_scan_bwd_params &q, cudaStream_t s) {
    static int staged_ok = -1;
    if (staged_ok < 0) { const char *e = getenv("ZG_SCAN_BWD_STAGED"); staged_ok = e ? atoi(e) : 1; }
    if (!scan_bwd_q4_fits(q)) return -1;
    const zg_scan_params &p = q.fwd;
    const int per_group = p.dim / p.ngroups;
    const long long nblk = (long long)p.ngroups * ((per_group + Q4_CH - 1) / Q4_CH) * p.batch;

    // staged variant: whole tiles and chunks, one layout for all activations, 16-byte aligned rows, 32-bit offsets
    constexpr int EPC = 16 / (int)sizeof(T);
    const bool has_z = p.z != nullptr;
    const bool tok = p.u_sd == 1 && p.delta_sd == 1 && q.dout_sd == 1 && q.du_sd == 1 && q.ddelta_sd == 1 && (!has_z || (p.z_sd == 1 && q.dz_sd == 1)) && p.dim > 1;
    const bool seq = !tok && p.u_sl == 1 && p.delta_sl == 1 && q.dout_sl == 1 && q.du_sl == 1 && q.ddelta_sl == 1 && (!has_z || (p.z_sl == 1 && q.dz_sl == 1)) && !p.z_rowmap;
    const bool bc_ok = (p.B_sn == 1 || p.B_sl == 1) && (p.C_sn == 1 || p.C_sl == 1);
    const uintptr_t al = reinterpret_cast<uintptr_t>(p.u) | reinterpret_cast<uintptr_t>(p.delta) | reinterpret_cast<uintptr_t>(p.z) | reinterpret_cast<uintptr_t>(q.dout) |
                         reinterpret_cast<uintptr_t>(p.B) | reinterpret_cast<uintptr_t>(p.C) | reinterpret_cast<uintptr_t>(q.du) | reinterpret_cast<uintptr_t>(q.ddelta) |
                         reinterpret_cast<uintptr_t>(q.dz);
    auto ok1 = [&](int64_t v) { return v == 1 || v % EPC == 0; };          // unit stride or whole 16-byte chunks
    bool strides_ok = ok1(p.u_sd) && ok1(p.u_sl) && ok1(p.delta_sd) && ok1(p.delta_sl) && ok1(q.dout_sd) && ok1(q.dout_sl) && ok1(q.du_sd) && ok1(q.du_sl) &&
                      ok1(q.ddelta_sd) && ok1(q.ddelta_sl) && ok1(p.B_sn) && ok1(p.B_sl) && ok1(p.C_sn) && ok1(p.C_sl) &&
                      p.u_sb % EPC == 0 && p.delta_sb % EPC == 0 && q.dout_sb % EPC == 0 && q.du_sb % EPC == 0 && q.ddelta_sb % EPC == 0 &&
                      p.B_sb % EPC == 0 && p.B_sg % EPC == 0 && p.C_sb % EPC == 0 && p.C_sg % EPC == 0;
    if (has_z) strides_ok = strides_ok && ok1(p.z_sd) && ok1(p.z_sl) && ok1(q.dz_sd) && ok1(q.dz_sl) && p.z_sb % EPC == 0 && q.dz_sb % EPC == 0;
    auto mag = [](int64_t v) { return v < 0 ? -v : v; };
    auto span = [&](int64_t sd, int64_t sl) { return (int64_t)p.dim * mag(sd) + (int64_t)p.seqlen * mag(sl); };
    const bool small = span(p.u_sd, p.u_sl) < 0x7fffffffLL && span(p.delta_sd, p.delta_sl) < 0x7fffffffLL && span(q.dout_sd, q.dout_sl) < 0x7fffffffLL &&
                       span(q.du_sd, q.du_sl) < 0x7fffffffLL && span(q.ddelta_sd, q.ddelta_sl) < 0x7fffffffLL &&
                       (!has_z || (span(p.z_sd, p.z_sl) < 0x7fffffffLL && span(q.dz_sd, q.dz_sl) < 0x7fffffffLL)) &&
                       16 * mag(p.B_sn) + (int64_t)p.seqlen * mag(p.B_sl) < 0x7fffffffLL && 16 * mag(p.C_sn) + (int64_t)p.seqlen * mag(p.C_sl) < 0x7fffffffLL;
    const bool staged = staged_ok && (tok || seq) && bc_ok && al % 16 == 0 && strides_ok && small && per_group % Q4_CH == 0 && p.seqlen % Q4_TS == 0 &&
                        p.u_sl >= 0 && p.u_sd >= 0;

    auto launch = [&](auto kern, int smem) -> int {
        cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (err != cudaSuccess) return zg_set_error("scan_bwd(q4): cudaFuncSetAttribute(%d B smem): %s", smem, cudaGetErrorString(err));
        cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        kern<<<(unsigned)nblk, Q4_THREADS, smem, s>>>(q);
        zg_count_launch();
        return zg_check_launch("scan_bwd(q4)");
    };
    if (staged) return launch(scan_bwd_q4_kernel<T, true, DET>, Q4Smem<T, true>::TOTAL);
    return launch(scan_bwd_q4_kernel<T, false, DET>, Q4Smem<T, false>::TOTAL);
}

}  // namespace zg
