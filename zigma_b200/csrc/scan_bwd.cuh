// Selective-scan (S6) backward for sm_90a -- same mapping as the forward (scan_fwd.cuh): a thread
// owns one channel, keeps dh / dA partial sums in registers and walks L in reverse, one 8-step chunk
// at a time (generic fallback: any dstate <= 64, constant (dim, dstate) B / C; the dstate == 16 input-dependent case runs
// scan_bwd_q4.cuh).  Replaces
// selective_scan_bwd_kernel (dis_mamba/csrc/selective_scan/selective_scan_bwd_kernel.cuh:75-489): no block-wide
// reverse scan, no BlockExchange.
//
// Per chunk: (1) the forward recurrence is recomputed from the checkpoint the forward kernel wrote at
// the chunk boundary (ckpt_every == 8), parking h_{l-1} of every step in shared memory
// ([step][state][thread]: conflict free); (2) the chunk is walked backwards:
//     dh_l = dy_l C_l + a_{l+1} dh_{l+1}            dC_l += dy_l h_l          dB_l += dh_l d_l u_l
//     du_l = dy_l D + d_l sum_n dh_l B_l             dA   += dh_l h_{l-1} a_l d_l
//     dd_l = sum_n dh_l (h_{l-1} a_l A + B_l u_l)    ddelta = dd_l * sigmoid(delta~)   (softplus')
//     dz_l = dout_l y_l sigmoid(z)(1 + z(1 - sigmoid(z)))      dD += dy_l u_l
// (selective_scan_bwd_kernel.cuh:186-213,252-296,439-452).  dB/dC are reduced over the 32 channels of
// a warp with a 31-shuffle transpose-reduce and added to the fp32 outputs with one atomic per
// (warp, state, step); dA/dD/ddelta_bias are accumulated over the whole row in registers and added
// once at the end (the reference uses fp32 atomics for all of these too, :297-316,467-488).
#pragma once
#include "zg_common.cuh"
#include "scan_bwd_q4.cuh"

namespace zg {

constexpr int BWD_CH = 64;
constexpr int BWD_TS = Q4_TS;   // == ckpt_every of the forward (8)

// CB: some of B / C is a constant (dim, dstate) weight (decided per operand at run time); false compiles the per-channel
// copies and accumulators away.
// DET: the gradient pointers of q address partial rows (zg_selective_scan_bwd_det): variable dB / dC one row per
// (channel tile within the group, warp), (2 tiles_per_group, batch, groups, dstate, seqlen); dA and constant dB / dC one
// row per batch row, (batch, dim, dstate); dD / d(delta_bias) (batch, dim).  Plain stores where the atomic path adds.
template <typename T, int NS, bool CB, bool DET>
__global__ void __launch_bounds__(BWD_CH) scan_bwd_kernel(const zg_scan_bwd_params q) {
    const zg_scan_params &p = q.fwd;
    constexpr int TS = BWD_TS, CH = BWD_CH;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float *hs = reinterpret_cast<float *>(smem_raw);        // [TS][NS][CH]  h_{l-1} per step
    float *bcf = hs + TS * NS * CH;                         // [TS][2*NS]    B | C as fp32

    const int tid = threadIdx.x, lane = tid & 31;
    const int E = p.dim, L = p.seqlen, N = p.dstate;
    const int per_group = E / p.ngroups;
    const int tiles_per_group = (per_group + CH - 1) / CH;
    const int tiles = tiles_per_group * p.ngroups;
    const int b = blockIdx.x / tiles;
    const int tile = blockIdx.x % tiles;
    const int g = tile / tiles_per_group;
    const int e0 = g * per_group + (tile % tiles_per_group) * CH;
    const int e_end = min(e0 + CH, (g + 1) * per_group);
    const bool active = e0 + tid < e_end;
    const int e = active ? e0 + tid : e0;                   // inactive threads shadow a valid channel
    const bool has_z = p.z != nullptr;
    const bool softplus = (p.flags & ZG_SCAN_DELTA_SOFTPLUS) != 0;
    // constant B / C (selective_scan.cpp:238-278: fp32 (dim, dstate) weights instead of (batch, groups, dstate, seqlen) inputs):
    // read per channel, their gradients accumulated per channel over the whole row (selective_scan_bwd_kernel.cuh:297-316)
    const bool varB = CB ? (p.flags & ZG_SCAN_VARIABLE_B) != 0 : true, varC = CB ? (p.flags & ZG_SCAN_VARIABLE_C) != 0 : true;

    const T *gu = reinterpret_cast<const T *>(p.u) + (int64_t)b * p.u_sb + (int64_t)e * p.u_sd;
    const T *gd = reinterpret_cast<const T *>(p.delta) + (int64_t)b * p.delta_sb + (int64_t)e * p.delta_sd;
    const T *gz = has_z ? reinterpret_cast<const T *>(p.z) + (int64_t)b * p.z_sb + (int64_t)e * p.z_sd : nullptr;
    const T *gdo = reinterpret_cast<const T *>(q.dout) + (int64_t)b * q.dout_sb + (int64_t)e * q.dout_sd;
    const T *gB = reinterpret_cast<const T *>(p.B) + (int64_t)b * p.B_sb + (int64_t)g * p.B_sg;
    const T *gC = reinterpret_cast<const T *>(p.C) + (int64_t)b * p.C_sb + (int64_t)g * p.C_sg;
    T *gdu = reinterpret_cast<T *>(q.du) + (int64_t)b * q.du_sb + (int64_t)e * q.du_sd;
    T *gdd = reinterpret_cast<T *>(q.ddelta) + (int64_t)b * q.ddelta_sb + (int64_t)e * q.ddelta_sd;
    T *gdz = has_z ? reinterpret_cast<T *>(q.dz) + (int64_t)b * q.dz_sb + (int64_t)e * q.dz_sd : nullptr;
    const int64_t det_row = DET ? (int64_t)((tile % tiles_per_group) * 2 + (tid >> 5)) * p.batch * p.ngroups * N * L : 0;
    float *gdB = q.dB + (varB ? det_row + ((int64_t)b * p.ngroups + g) * (int64_t)N * L : 0);     // (batch, groups, dstate, seqlen) contiguous
    float *gdC = q.dC + (varC ? det_row + ((int64_t)b * p.ngroups + g) * (int64_t)N * L : 0);
    const int nck = (L + TS - 1) / TS;
    const float *ck = p.ckpt + ((int64_t)b * nck * E + e) * (int64_t)N;     // (batch, n_ckpt, dim, dstate)

    float A[NS], dA[NS], dh[NS], a_next[NS], Bc[NS], Cc[NS], dBc[NS], dCc[NS];
#pragma unroll
    for (int n = 0; n < NS; ++n) {
        A[n] = (n < N) ? p.A[(int64_t)e * N + n] : 0.f;
        Bc[n] = (!varB && n < N) ? reinterpret_cast<const float *>(p.B)[(int64_t)e * N + n] : 0.f;
        Cc[n] = (!varC && n < N) ? reinterpret_cast<const float *>(p.C)[(int64_t)e * N + n] : 0.f;
        dA[n] = 0.f; dh[n] = 0.f; a_next[n] = 0.f; dBc[n] = 0.f; dCc[n] = 0.f;
    }
    const float Dv = p.D ? p.D[e] : 0.f;
    const float bias = p.delta_bias ? p.delta_bias[e] : 0.f;
    float dD_acc = 0.f, dbias_acc = 0.f;

    for (int k = nck - 1; k >= 0; --k) {
        const int l0 = k * TS;
        const int nsteps = min(TS, L - l0);
        __syncthreads();     // previous chunk done with bcf / hs
        for (int it = tid; it < 2 * TS * NS; it += CH) {
            const int w = it / (TS * NS), rem = it % (TS * NS);
            const int n = rem / TS, t = rem % TS;
            float v = 0.f;
            if (n < N && t < nsteps && (w == 0 ? varB : varC)) v = zg_to_float<T>(w == 0 ? gB[(int64_t)n * p.B_sn + l0 + t] : gC[(int64_t)n * p.C_sn + l0 + t]);
            bcf[t * 2 * NS + w * NS + n] = v;
        }
        __syncthreads();

        // ---- (1) forward recompute from the chunk-boundary checkpoint ----------------------------
        float dl[TS], uu[TS];
        float h[NS];
#pragma unroll
        for (int n = 0; n < NS; ++n) h[n] = (k > 0 && n < N) ? ck[(int64_t)(k - 1) * E * N + n] : 0.f;
#pragma unroll
        for (int t = 0; t < TS; ++t) {
            if (t < nsteps) {
                float d = zg_to_float<T>(gd[l0 + t]) + bias;
                if (softplus) d = zg_softplus20(d);
                dl[t] = d;
                uu[t] = zg_to_float<T>(gu[l0 + t]);
                const float du_ = d * uu[t];
#pragma unroll
                for (int n = 0; n < NS; ++n) {
                    hs[(t * NS + n) * CH + tid] = h[n];
                    h[n] = fmaf(zg_ex2(d * A[n] * ZG_LOG2E), h[n], du_ * (varB ? bcf[t * 2 * NS + n] : Bc[n]));
                }
            } else {
                dl[t] = 0.f; uu[t] = 0.f;
            }
        }

        // ---- (2) reverse sweep over the chunk ---------------------------------------------------------
#pragma unroll
        for (int t = TS - 1; t >= 0; --t) {
            if (t < nsteps) {       // uniform across the CTA
                const int l = l0 + t;
                const float d = dl[t], u_ = uu[t];
                float dout = active ? zg_to_float<T>(gdo[l]) : 0.f;
                float zz = 0.f, sg = 0.f, dy = dout;
                if (has_z) {
                    zz = zg_to_float<T>(gz[l]);
                    sg = 1.f / (1.f + __expf(-zz));
                    dy = dout * zz * sg;
                }
                dD_acc += dy * u_;
                float du_ = dy * Dv, dd = 0.f, y = Dv * u_;
                float red[2 * NS];     // [0, NS): dB   [NS, 2NS): dC   (this thread's contribution)
#pragma unroll
                for (int n = 0; n < NS; ++n) {
                    const float Bn = varB ? bcf[t * 2 * NS + n] : Bc[n], Cn = varC ? bcf[t * 2 * NS + NS + n] : Cc[n];
                    const float a = zg_ex2(d * A[n] * ZG_LOG2E);
                    const float hprev = hs[(t * NS + n) * CH + tid];
                    const float hl = fmaf(a, hprev, d * u_ * Bn);
                    y = fmaf(Cn, hl, y);
                    const float dhn = fmaf(a_next[n], dh[n], dy * Cn);
                    dh[n] = dhn;
                    a_next[n] = a;
                    const float da = dhn * hprev * a;         // d/d(d*A) of the a*h_{l-1} term
                    dd = fmaf(da, A[n], dd);
                    dd = fmaf(dhn * Bn, u_, dd);
                    dA[n] = fmaf(da, d, dA[n]);
                    du_ = fmaf(dhn * d, Bn, du_);
                    red[n] = dhn * d * u_;
                    red[NS + n] = dy * hl;
                }
                if (softplus) dd *= zg_softplus_grad(d);     // sigmoid(delta~) = 1 - exp(-softplus(delta~))
                dbias_acc += dd;
                if (active) {
                    gdu[l] = zg_from_float<T>(du_);
                    gdd[l] = zg_from_float<T>(dd);
                    if (has_z) gdz[l] = zg_from_float<T>(dout * y * sg * (1.f + zz * (1.f - sg)));
                }
                if (!varB || !varC) {      // constant operand: its gradient stays with the channel
#pragma unroll
                    for (int n = 0; n < NS; ++n) {
                        if (!varB) dBc[n] += red[n];
                        if (!varC) dCc[n] += red[NS + n];
                    }
                }
                // transpose-reduce the 2*NS per-thread values over the 32 lanes of the warp:
                // afterwards lane i (i < 2*NS) holds the warp total of value i.
                if (!varB && !varC) {
                    // nothing to reduce across channels
                } else if (NS > 16) {      // wide states: one warp sum per value (a fallback, not a fast path)
#pragma unroll
                    for (int j = 0; j < 2 * NS; ++j) {
                        const float tot = zg_warp_sum(red[j]);
                        const int n = j < NS ? j : j - NS;
                        if (lane == 0 && n < N && (j < NS ? varB : varC)) {
                            if constexpr (DET) (j < NS ? gdB : gdC)[(int64_t)n * L + l] = tot;
                            else atomicAdd((j < NS ? gdB : gdC) + (int64_t)n * L + l, tot);
                        }
                    }
                } else if (NS == 16) {
#pragma unroll
                    for (int half = 16; half >= 1; half >>= 1) {
                        const bool up = (lane & half) != 0;
#pragma unroll
                        for (int j = 0; j < half; ++j) {
                            const float send = up ? red[j] : red[j + half];
                            const float keep = up ? red[j + half] : red[j];
                            red[j] = keep + __shfl_xor_sync(0xffffffffu, send, half);
                        }
                    }
                    float *dst = (lane < NS) ? gdB + (int64_t)lane * L + l : gdC + (int64_t)(lane - NS) * L + l;
                    if ((lane < NS ? lane : lane - NS) < N && (lane < NS ? varB : varC)) {
                        if constexpr (DET) *dst = red[0];
                        else atomicAdd(dst, red[0]);
                    }
                } else {   // NS == 8: 16 values -> first fold the two half-warps, then transpose-reduce over 16 lanes
#pragma unroll
                    for (int j = 0; j < 2 * NS; ++j) red[j] += __shfl_xor_sync(0xffffffffu, red[j], 16);
#pragma unroll
                    for (int half = 8; half >= 1; half >>= 1) {
                        const bool up = (lane & half) != 0;
#pragma unroll
                        for (int j = 0; j < half; ++j) {
                            const float send = up ? red[j] : red[j + half];
                            const float keep = up ? red[j + half] : red[j];
                            red[j] = keep + __shfl_xor_sync(0xffffffffu, send, half);
                        }
                    }
                    const int v = lane & 15;
                    if (lane < 16) {
                        float *dst = (v < NS) ? gdB + (int64_t)v * L + l : gdC + (int64_t)(v - NS) * L + l;
                        if ((v < NS ? v : v - NS) < N && (v < NS ? varB : varC)) {
                            if constexpr (DET) *dst = red[0];
                            else atomicAdd(dst, red[0]);
                        }
                    }
                }
            }
        }
    }
    if (DET && active) {
        const int64_t be = (int64_t)b * E + e;
#pragma unroll
        for (int n = 0; n < NS; ++n)
            if (n < N) {
                q.dA[be * N + n] = dA[n];
                if (!varB) q.dB[be * N + n] = dBc[n];
                if (!varC) q.dC[be * N + n] = dCc[n];
            }
        if (q.dD) q.dD[be] = dD_acc;
        if (q.ddelta_bias) q.ddelta_bias[be] = dbias_acc;
    } else if (active) {
#pragma unroll
        for (int n = 0; n < NS; ++n)
            if (n < N) {
                atomicAdd(q.dA + (int64_t)e * N + n, dA[n]);
                if (!varB) atomicAdd(q.dB + (int64_t)e * N + n, dBc[n]);      // (dim, dstate) fp32
                if (!varC) atomicAdd(q.dC + (int64_t)e * N + n, dCc[n]);
            }
        if (q.dD) atomicAdd(q.dD + e, dD_acc);
        if (q.ddelta_bias) atomicAdd(q.ddelta_bias + e, dbias_acc);
    }
}

template <typename T, int NS, bool DET, bool CB = false> static int launch_scan_bwd(const zg_scan_bwd_params &q, cudaStream_t s) {
    const zg_scan_params &p = q.fwd;
    if constexpr (!CB) {
        if (!(p.flags & ZG_SCAN_VARIABLE_B) || !(p.flags & ZG_SCAN_VARIABLE_C)) return launch_scan_bwd<T, NS, DET, true>(q, s);
    }
    const int per_group = p.dim / p.ngroups;
    const int tiles = p.ngroups * ((per_group + BWD_CH - 1) / BWD_CH);
    const int smem = (BWD_TS * NS * BWD_CH + BWD_TS * 2 * NS) * (int)sizeof(float);
    auto kern = scan_bwd_kernel<T, NS, CB, DET>;
    cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (err != cudaSuccess) return zg_set_error("scan_bwd: cudaFuncSetAttribute(%d B smem): %s", smem, cudaGetErrorString(err));
    const long long nblk = (long long)tiles * p.batch;
    if (nblk > 0x7fffffffLL) return zg_set_error("scan_bwd: grid too large");
    kern<<<(unsigned)nblk, BWD_CH, smem, s>>>(q);
    zg_count_launch();
    return zg_check_launch("scan_bwd");
}

template <typename T, bool DET> static int scan_bwd_t(const zg_scan_bwd_params &q, cudaStream_t s) {
    const int rc = try_launch_scan_bwd_q4<T, DET>(q, s);
    if (rc >= 0) return rc;
    {   // generic kernel: one thread per channel walking its own row
        const zg_scan_params &p = q.fwd;
        ZG_REQUIRE(p.z_rowmap == nullptr, "selective_scan_bwd: z_rowmap needs the dstate == 16 kernel");
    ZG_REQUIRE(p.u_sl == 1 && p.delta_sl == 1 && q.dout_sl == 1 && q.du_sl == 1 && q.ddelta_sl == 1 && (!p.z || (p.z_sl == 1 && q.dz && q.dz_sl == 1)) &&
                   (!(p.flags & ZG_SCAN_VARIABLE_B) || p.B_sl == 1 || p.seqlen == 1) && (!(p.flags & ZG_SCAN_VARIABLE_C) || p.C_sl == 1 || p.seqlen == 1),
               "selective_scan_bwd: the generic kernel (dstate != 16) needs seq-contiguous tensors");
    }
    if (q.fwd.dstate <= 8) return launch_scan_bwd<T, 8, DET>(q, s);
    if (q.fwd.dstate <= 16) return launch_scan_bwd<T, 16, DET>(q, s);
    if (q.fwd.dstate <= 32) return launch_scan_bwd<T, 32, DET>(q, s);
    if (q.fwd.dstate <= 64) return launch_scan_bwd<T, 64, DET>(q, s);      // (register-heavy: the state arrays spill; correctness fallback)
    return zg_set_error("selective_scan_bwd: dstate <= 64 supported (like the forward), got %d", q.fwd.dstate);
}

}  // namespace zg

// one instantiation per translation unit: scan_bwd.cu (atomic path), scan_bwd_det.cu (DET) -- the two compile in parallel
template <bool DET> static int scan_bwd_dispatch(const zg_scan_bwd_params &q, cudaStream_t s) {
    switch (q.fwd.dtype) {
        case ZG_F32: return zg::scan_bwd_t<float, DET>(q, s);
        case ZG_F16: return zg::scan_bwd_t<__half, DET>(q, s);
        default: return zg::scan_bwd_t<__nv_bfloat16, DET>(q, s);
    }
}
int zg_scan_bwd_launch_det(const zg_scan_bwd_params &q, cudaStream_t s);      // scan_bwd_det.cu
