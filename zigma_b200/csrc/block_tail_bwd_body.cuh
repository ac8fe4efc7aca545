// Body of block_tail_bwd_kernel and block_tail_dp_bwd_kernel (norm.cu), included inside each kernel.  The including kernel
// defines T, MAXQ, DET (template arguments), DP (constexpr bool), p (const zg_block_tail_bwd_params) and path_scale.
// A __device__ function would do the same job, but inlining it changes the register allocation of the MAXQ = 8 DET
// instantiations, which spill, so the plain kernels would no longer compile to the code they had before DP existed.
    // per-batch column sums live in shared memory (lane-private slots, no conflicts): keeping all four accumulator sets
    // in registers cost 212 registers = 8 warps per SM, too few for a streaming kernel
    extern __shared__ __align__(16) float tailb_smem[];
    float4 *acc_s = reinterpret_cast<float4 *>(tailb_smem) + (threadIdx.x >> 5) * (3 * MAXQ * 32) + (threadIdx.x & 31);   // [warp][3][MAXQ][32 lanes]
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int lane = threadIdx.x & 31;
    const int64_t nrows = (int64_t)p.batch * p.seqlen;
    // persistent warps, contiguous partition: warp i owns rows [i * per, (i + 1) * per) -- equal work for every warp and at
    // most one batch boundary inside a range, so the per-batch sums are flushed once or twice per warp
    const int64_t per = (nrows + nwarps - 1) / nwarps;
    const int D = p.dim, nq = D >> 2;
    const float invD = 1.f / D;
    const T *nw = reinterpret_cast<const T *>(p.norm_w);
    float w[MAXQ][4], acc_w[MAXQ][4];
#pragma unroll
    for (int k = 0; k < MAXQ; ++k) {
        const int q = lane + 32 * k;
        if (q < nq) ld4<T>(nw, 4 * q, w[k]);
#pragma unroll
        for (int i = 0; i < 4; ++i) acc_w[k][i] = 0.f;
#pragma unroll
        for (int j = 0; j < 3; ++j) acc_s[(j * MAXQ + k) * 32] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
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
    if (row0 < row1) {
    int cur_b = (int)(row0 / p.seqlen);
    for (int64_t row = row0; row < row1; ++row) {
        const int b = (int)(row / p.seqlen), l = (int)(row % p.seqlen);
        if (b != cur_b) { flush_batch(cur_b); cur_b = b; }
        const int64_t mrow = (int64_t)b * p.seqlen + (p.rowmap ? p.rowmap[l] : l);
        const float *r = p.r + row * D;
        const T *dn = p.d_normed ? reinterpret_cast<const T *>(p.d_normed) + row * D : nullptr;
        const T *dm = p.d_modded ? reinterpret_cast<const T *>(p.d_modded) + row * D : nullptr;
        const float *dro = p.d_residual_out ? p.d_residual_out + row * D : nullptr;
        const T *mix = p.mix ? reinterpret_cast<const T *>(p.mix) + mrow * D : nullptr;
        const T *gate = p.gate ? reinterpret_cast<const T *>(p.gate) + (int64_t)b * p.mod_rs : nullptr;
        const T *scale = p.scale ? reinterpret_cast<const T *>(p.scale) + (int64_t)b * p.mod_rs : nullptr;
        const float rstd = p.rstd[row];
        [[maybe_unused]] float dps = 1.f;
        if constexpr (DP) dps = zg_to_float<T>(reinterpret_cast<const T *>(path_scale)[b]);
        // ---- all streaming loads of the row first ----
        float4 rr[MAXQ];
        Raw4<T> rdn[MAXQ], rdm[MAXQ], rmx[MAXQ];
#pragma unroll
        for (int k = 0; k < MAXQ; ++k) {
            const int q = lane + 32 * k;
            if (q < nq) {
                rr[k] = *reinterpret_cast<const float4 *>(r + 4 * q);
                if (dn) rdn[k] = ldraw<T>(dn, 4 * q);
                if (dm) rdm[k] = ldraw<T>(dm, 4 * q);
                if (mix) rmx[k] = ldraw<T>(mix, 4 * q);
            }
        }
        // ---- dy, per-column sums, c1 = mean(xhat * w * dy)  (xhat = r * rstd is recomputed where needed: registers) ----
        float dy[MAXQ][4];
        float c1 = 0.f;
#pragma unroll
        for (int k = 0; k < MAXQ; ++k) {
            const int q = lane + 32 * k;
            if (q < nq) {
                const float xh[4] = {rr[k].x * rstd, rr[k].y * rstd, rr[k].z * rstd, rr[k].w * rstd};
                float a[4] = {0.f, 0.f, 0.f, 0.f};
                if (dn) cvt4<T>(rdn[k], a);
                if (dm) {
                    float sc[4], m[4];
                    cvt4<T>(rdm[k], m);
                    ld4<T>(scale, 4 * q, sc);
                    float4 ash = acc_s[(1 * MAXQ + k) * 32], asc = acc_s[(2 * MAXQ + k) * 32];
                    float *psh = &ash.x, *psc = &asc.x;
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        a[i] = fmaf(m[i], 1.f + sc[i], a[i]);
                        psh[i] += m[i];
                        psc[i] = fmaf(m[i], xh[i] * w[k][i], psc[i]);       // d_modded * normed
                    }
                    acc_s[(1 * MAXQ + k) * 32] = ash; acc_s[(2 * MAXQ + k) * 32] = asc;
                }
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    dy[k][i] = a[i];
                    acc_w[k][i] = fmaf(a[i], xh[i], acc_w[k][i]);
                    c1 = fmaf(xh[i], a[i] * w[k][i], c1);
                }
            }
        }
        c1 = zg_warp_sum(c1) * invD;
        // ---- dr, outputs ----
        float *drin = p.d_residual_in ? p.d_residual_in + row * D : nullptr;
        T *dx = reinterpret_cast<T *>(p.d_x) + row * D;
        T *dmix = p.d_mix ? reinterpret_cast<T *>(p.d_mix) + mrow * D : nullptr;
#pragma unroll
        for (int k = 0; k < MAXQ; ++k) {
            const int q = lane + 32 * k;
            if (q < nq) {
                const float xh[4] = {rr[k].x * rstd, rr[k].y * rstd, rr[k].z * rstd, rr[k].w * rstd};
                float dr[4], dh[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) dr[i] = (dy[k][i] * w[k][i] - xh[i] * c1) * rstd;
                if (dro) {
                    const float4 t = *reinterpret_cast<const float4 *>(dro + 4 * q);
                    dr[0] += t.x; dr[1] += t.y; dr[2] += t.z; dr[3] += t.w;
                }
                if (drin) st4<float>(drin, 4 * q, dr);
#pragma unroll
                for (int i = 0; i < 4; ++i) dh[i] = round_to<T>(dr[i]);
                if constexpr (DP) {
#pragma unroll
                    for (int i = 0; i < 4; ++i) dh[i] = round_to<T>(__fmul_rn(dh[i], dps));
                }
                st4<T>(dx, 4 * q, dh);
                if (mix) {
                    float m[4], g[4], o[4];
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
    }
    flush_batch(cur_b);
    }
    // d_norm_w: sum over the CTA's 4 warps in shared memory, then ONE plain store per column into this CTA's row of the
    // (gridDim.x, dim) partials buffer -- atomics from every warp onto the same 640 addresses serialised for ~50 us
    // (first version, 126 us per call); the caller adds the few hundred partial rows up.
    if (p.d_norm_w) {
        __syncthreads();
        float *red = tailb_smem;                           // [4][4 * 32 * MAXQ]
#pragma unroll
        for (int k = 0; k < MAXQ; ++k)
            *reinterpret_cast<float4 *>(red + (threadIdx.x >> 5) * (128 * MAXQ) + 4 * (lane + 32 * k)) = make_float4(acc_w[k][0], acc_w[k][1], acc_w[k][2], acc_w[k][3]);
        __syncthreads();
        for (int c = threadIdx.x; c < D; c += 128)
            p.d_norm_w[(int64_t)blockIdx.x * D + c] = red[c] + red[128 * MAXQ + c] + red[2 * 128 * MAXQ + c] + red[3 * 128 * MAXQ + c];
    }
