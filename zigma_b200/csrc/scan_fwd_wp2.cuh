// Selective-scan forward, warp-private pipeline with TWO channels per lane (32 channels x 16 states per warp).
//
// Why: ncu of both hot-path kernels shows a second resource next to the MUFU pipe: the
// shared-memory data pipe of the SM runs 55 % (CTA-wide kernel) / 72 % (warp-private, one channel per lane) of its wavefront
// peak, three quarters of it the B / C rows of the recurrence: every lane fetches its eight B and eight C values per step
// (4 LDS.128 = 2048 lane-bytes = 8 wavefronts per warp-step, broadcast or not), and those loads share the sub-partition's MIO
// queue with the MUFU instructions, so a queue head that waits for the (SM-wide) data pipe also holds back the exponentials
// behind it (stall `mio_throttle` 2.9-3.1 warps per issue while the MUFU pipe idles a quarter of the time).  With two channels
// per lane the same B / C registers feed twice the recurrences: 11 wavefronts per 32 channel-steps instead of 20.6, 3 shared
// loads + 1 store per lane-step instead of 2 x (5 + 1), half the B|C staging / conversion per channel, and ~12 % fewer issued
// instructions per (b, e, l).  Price: ~100 registers, half the warps (4.3 per sub-partition at config 2), each with twice the
// independent work (16 MUFU back to back per step).
//
// Everything else is scan_fwd_wp.cuh: a warp stages its own u / delta / z / B|C rows (8 steps per stage, 3-deep ring, one
// mbarrier per slot, 16-byte cp.async chunks, or TMA tiles for u / delta), no block barrier.  Per channel the operations and
// their order are those of scan_fwd_tma_kernel: results are bit-identical.
// Semantics: selective_scan_fwd_kernel.cuh:153-171, :216-261, :280-298.
#pragma once
#include "scan_fwd_wp.cuh"

namespace zg {

constexpr int WP2_CH = 32;            // channels per warp
constexpr int WP2_MAX_WARPS = 9;      // 288 threads x 2 CTAs per SM: 112 registers per thread

struct Wp2Layout {                    // per warp
    static constexpr int NSTAGE = 3;
    static constexpr int TILE = PT_TL * WP2_CH * 2;               // 8 steps x 64 B
    static constexpr int RAW = 3 * TILE + PT_TL * 64;             // u | delta | z | B|C rows (64 B each)
    static constexpr int DDU_ROW = WP2_CH * 8;                    // (delta', delta' u) fp32 pairs of one step
    static constexpr int DDU_OFF = NSTAGE * RAW;
    static constexpr int BCF_OFF = DDU_OFF + PT_TL * DDU_ROW;     // fp32 B / C values, see bc_convert
    static constexpr int BAR_OFF = BCF_OFF + PT_TL * 32 * 4;
    static constexpr int WARP_BYTES = ((BAR_OFF + NSTAGE * 8 + 127) / 128) * 128;
};

// one stage (8 steps) of the recurrence for the lane's two channels x 8 states.
// ddu_j: the (delta', delta' u) pairs of the two channels (16 bytes per step, pitch PITCH); bq: the lane's B / C quads
// (bc_convert layout: step t at + 16 t floats; B quad k at + 128 k, C quad k at + 8 + 128 k floats); ypart: where the lane's two
// partial sums of a step go (8 bytes: the lower or the upper half of the 16 bytes the pairs came from).
// Software-pipelined like pt_main_stage: the 16 decay factors of step t + 1 are issued before the FMAs of step t.
template <int PITCH>
__device__ __forceinline__ void wp2_main_stage(const unsigned char *__restrict__ ddu_j, const float *__restrict__ bq, unsigned char *__restrict__ ypart,
                                               zg_f2 (&h)[2][4], const zg_f2 (&Al)[2][4], int sync_step = -1, int bar_threads = 0) {
    auto decay = [&](float dlx, const zg_f2 (&al)[4], zg_f2 (&a)[4]) {
        const zg_f2 dl = zg_splat2(dlx);
#pragma unroll
        for (int q = 0; q < 4; ++q) a[q] = zg_ex2_mufu2(zg_mul2(dl, al[q]));
    };
    zg_f2 a0[4], a1[4];
    float4 dd = *reinterpret_cast<const float4 *>(ddu_j);          // (delta'0, delta'0 u0, delta'1, delta'1 u1)
    decay(dd.x, Al[0], a0);
    decay(dd.z, Al[1], a1);
#pragma unroll
    for (int t = 0; t < PT_TL; ++t) {
        const float4 *bc = reinterpret_cast<const float4 *>(bq + t * 16);
        zg_f2 Bp[4], Cp[4];
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const float4 Bk = bc[32 * k], Ck = bc[2 + 32 * k];
            Bp[2 * k] = make_float2(Bk.x, Bk.y); Bp[2 * k + 1] = make_float2(Bk.z, Bk.w);
            Cp[2 * k] = make_float2(Ck.x, Ck.y); Cp[2 * k + 1] = make_float2(Ck.z, Ck.w);
        }
        const zg_f2 du0 = zg_splat2(dd.y), du1 = zg_splat2(dd.w);
        zg_f2 n0[4], n1[4];
        if (t + 1 < PT_TL) {                                       // next step's pairs and decays: in flight during this step's FMAs
            dd = *reinterpret_cast<const float4 *>(ddu_j + (t + 1) * PITCH);
            decay(dd.x, Al[0], n0);
            decay(dd.z, Al[1], n1);
        }
        zg_f2 y0 = zg_splat2(0.f), y1 = zg_splat2(0.f);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            h[0][q] = zg_fma2(a0[q], h[0][q], zg_mul2(du0, Bp[q]));
            y0 = zg_fma2(Cp[q], h[0][q], y0);
            h[1][q] = zg_fma2(a1[q], h[1][q], zg_mul2(du1, Bp[q]));
            y1 = zg_fma2(Cp[q], h[1][q], y1);
        }
        // (both lanes of the channel pair have read the 16 bytes -- one converged LDS -- before either overwrites its half)
        *reinterpret_cast<float2 *>(ypart + t * PITCH) = make_float2(y0.x + y0.y, y1.x + y1.y);
        if (t == sync_step) asm volatile("bar.sync 1, %0;" ::"r"(bar_threads) : "memory");      // staggered fairness barrier, see wp_body
        if (t + 1 < PT_TL) {
#pragma unroll
            for (int q = 0; q < 4; ++q) { a0[q] = n0[q]; a1[q] = n1[q]; }
        }
    }
}

// The work of one warp: 32 channels [e0, e0 + 32) of group g of batch row b, all seqlen steps.  `smem`: the warp's Wp2Layout bytes.
template <typename T, bool CKPT, bool PLAIN, bool TMA>
__device__ __forceinline__ void wp2_body(const zg_scan_params &p, const PtMaps &maps, unsigned char *smem, const int lane, const int b, const int g, const int e0,
                                         const int sync_every = 0, const int cta_warps = 0, const int sync_step = 0) {
    static_assert(sizeof(T) == 2, "16-bit I/O only");
    using LY = Wp2Layout;
    constexpr int NSTAGE = LY::NSTAGE, TL = PT_TL, TILE = LY::TILE, NITEM = 4;
    unsigned char *ddu = smem + LY::DDU_OFF;
    float *bcf = reinterpret_cast<float *>(smem + LY::BCF_OFF);
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + LY::BAR_OFF);

    const int part = lane & 1;                                     // which 8 states of the lane's two channels
    const int E = p.dim, L = p.seqlen;
    const int e = e0 + (lane >> 1) * 2;                            // main phase: this lane's first channel (the second is e + 1)
    const bool has_z = PLAIN ? true : (p.z != nullptr);
    const bool softplus = PLAIN ? true : ((p.flags & ZG_SCAN_DELTA_SOFTPLUS) != 0);
    const int nstages = L / TL;
    int sync_left = sync_every;

    // ---- per-thread constants -----------------------------------------------------------------------------------
    zg_f2 Al2p[2][4], h2[2][4];
#pragma unroll
    for (int c = 0; c < 2; ++c)
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float2 a = *reinterpret_cast<const float2 *>(p.A + (int64_t)(e + c) * 16 + 8 * part + 2 * k);
            Al2p[c][k] = zg_mul2(a, zg_splat2(ZG_LOG2E));
            h2[c][k] = zg_splat2(0.f);
        }
    // pre / post items of a lane: channel pair lane % 16 at steps lane / 16 + 2 k, k = 0..3 (the same items in both phases:
    // post reads the partial y from the 16 bytes its own pre filled)
    const int pair = lane & 15, r0 = lane >> 4;
    const int it_raw = r0 * 64 + pair * 4;                         // byte offset in a 8 x 64 B tile; item k: + 128 k
    const int it_ddu = r0 * LY::DDU_ROW + pair * 16;               // item k: + 2 k rows
    const float2 Dv = p.D ? *reinterpret_cast<const float2 *>(p.D + e0 + 2 * pair) : make_float2(0.f, 0.f);
    const float2 biasv = p.delta_bias ? *reinterpret_cast<const float2 *>(p.delta_bias + e0 + 2 * pair) : make_float2(0.f, 0.f);

    if (lane == 0) {        // full[s]: one cp.async arrival per lane and stage (+ the TMA issuer's expect_tx)
#pragma unroll
        for (int s = 0; s < NSTAGE; ++s) zg_mbar_init(&full[s], TMA ? 33 : 32);
        zg_mbar_fence_init();
    }
    __syncwarp();

    // ---- producer side of the lane: one 16-byte chunk of each of the four tiles -----------------------------------
    // B|C rows: chunk `lane` = step lane / 4, B or C, which 16 bytes
    const unsigned char *bc_src;
    uint32_t bc_step;
    {
        const int r = lane >> 2, w = (lane >> 1) & 1, j = lane & 1;
        const T *src = w ? reinterpret_cast<const T *>(p.C) + (int64_t)b * p.C_sb + (int64_t)g * p.C_sg + (int64_t)r * p.C_sl
                         : reinterpret_cast<const T *>(p.B) + (int64_t)b * p.B_sb + (int64_t)g * p.B_sg + (int64_t)r * p.B_sl;
        bc_src = reinterpret_cast<const unsigned char *>(src + j * 8);
        bc_step = (uint32_t)(w ? p.C_sl : p.B_sl) * (2u * TL);
    }
    // u / delta / z: row lane / 4 of the stage, 16-byte quarter lane % 4; the z row goes through z_rowmap when given.
    // batch element b of z: plain batch stride, or two-level (b / K, b % K) for the temporal video scan (zg_scan_params.z_batch_inner)
    const int zr = lane >> 2, zj = lane & 3;
    const int64_t z_boff = p.z_batch_inner > 0 ? (int64_t)(b / p.z_batch_inner) * p.z_sb + (int64_t)(b % p.z_batch_inner) * p.z_sbi : (int64_t)b * p.z_sb;
    const unsigned char *zsrc = has_z ? reinterpret_cast<const unsigned char *>(reinterpret_cast<const T *>(p.z) + z_boff + e0 + zj * 8) : nullptr;
    const uint32_t z_sl2 = (uint32_t)p.z_sl * 2u;                  // byte offsets inside a batch element fit 32 bits (host check)
    const int32_t *zmap = p.z_rowmap;
    int zrow_next = has_z ? (zmap ? zmap[zr] : zr) : 0;            // (permuted) source row of the NEXT stage to issue
    const unsigned char *u_src = nullptr, *d_src = nullptr;
    uint32_t u_step = 0, d_step = 0;
    if constexpr (!TMA) {
        u_src = reinterpret_cast<const unsigned char *>(reinterpret_cast<const T *>(p.u) + (int64_t)b * p.u_sb + (int64_t)zr * p.u_sl + e0 + zj * 8);
        d_src = reinterpret_cast<const unsigned char *>(reinterpret_cast<const T *>(p.delta) + (int64_t)b * p.delta_sb + (int64_t)zr * p.delta_sl + e0 + zj * 8);
        u_step = (uint32_t)p.u_sl * (2u * TL);
        d_step = (uint32_t)p.delta_sl * (2u * TL);
    }
    int s_issue = 0;                                               // stages are issued in order
    auto issue_stage = [&](int slot) {                             // all lanes
        if (s_issue >= nstages) return;
        unsigned char *raw = smem + slot * LY::RAW;
        uint64_t *bar = &full[slot];
        const int l0 = s_issue * TL;
        if constexpr (TMA) {
            if (lane == 0) {
                zg_mbar_expect_tx(bar, 2 * TILE);
                pt_tma_load_3d(raw, &maps.u, bar, e0, l0, b);
                pt_tma_load_3d(raw + TILE, &maps.d, bar, e0, l0, b);
            }
        } else {
            zg_cp_async16(raw + lane * 16, u_src);
            zg_cp_async16(raw + TILE + lane * 16, d_src);
            u_src += u_step;
            d_src += d_step;
        }
        if (has_z) {
            zg_cp_async16(raw + 2 * TILE + lane * 16, zsrc + (uint32_t)zrow_next * z_sl2);
            const int ln = l0 + TL + zr;
            zrow_next = (ln < L) ? (zmap ? zmap[ln] : ln) : 0;
        }
        zg_cp_async16(raw + 3 * TILE + lane * 16, bc_src);
        bc_src += bc_step;
        pt_cp_async_arrive(bar);
        ++s_issue;
    };
#pragma unroll
    for (int s = 0; s < NSTAGE; ++s) issue_stage(s);

    // ---- pre / post work of a lane's four items -------------------------------------------------------------------
    // B | C rows -> fp32.  Lane c converts chunk c (step c / 4; B or C; states 8 j .. 8 j + 7) and writes its first four values
    // to quad c of region 0 and the last four to quad c of region 1 (two conflict-free STS.128).  The lane of the main phase
    // with state half `part` then finds, for step t: B quads at 16 t + 4 part (+ 128 k), C quads at 16 t + 8 + 4 part (+ 128 k).
    auto bc_convert = [&](const unsigned char *raw) {
        const uint4 v = *reinterpret_cast<const uint4 *>(raw + 3 * TILE + lane * 16);
        const float2 a = pt_unpack2<T>(v.x), c = pt_unpack2<T>(v.y), d = pt_unpack2<T>(v.z), f = pt_unpack2<T>(v.w);
        float4 *dst = reinterpret_cast<float4 *>(bcf) + lane;
        dst[0] = make_float4(a.x, a.y, c.x, c.y);
        dst[32] = make_float4(d.x, d.y, f.x, f.y);
    };
    auto pre_item = [&](int k, const unsigned char *raw) {         // bias, softplus, * u -> (delta', delta' u) pairs
        float2 dl = pt_unpack2<T>(*reinterpret_cast<const uint32_t *>(raw + TILE + it_raw + k * 128));
        dl = zg_add2(dl, biasv);
        if (softplus) dl = pt_softplus20_2(dl);
        const float2 du = zg_mul2(dl, pt_unpack2<T>(*reinterpret_cast<const uint32_t *>(raw + it_raw + k * 128)));
        *reinterpret_cast<float4 *>(ddu + it_ddu + k * 2 * LY::DDU_ROW) = make_float4(dl.x, du.x, dl.y, du.y);
    };
    // output rows: step l -> sequence position l, or seqlen - 1 - l (ZG_SCAN_OUT_REVERSE: the backward sweep of scan_type v2)
    const bool out_rev = PLAIN ? false : ((p.flags & ZG_SCAN_OUT_REVERSE) != 0), out_acc = PLAIN ? false : ((p.flags & ZG_SCAN_OUT_ACCUMULATE) != 0);
    const int64_t out_row = out_rev ? -p.out_sl : p.out_sl;
    T *gout = reinterpret_cast<T *>(p.out) + (int64_t)b * p.out_sb + (int64_t)(out_rev ? L - 1 - r0 : r0) * p.out_sl + e0 + 2 * pair;
    const int64_t out_item = 2 * out_row, out_stage = (int64_t)TL * out_row;
    auto post_item = [&](int k, const unsigned char *raw) {        // y = y_lo + y_hi + D u, SiLU(z) gate, store
        // the main phase left (lo of channel 0, lo of channel 1, hi of channel 0, hi of channel 1) in the pair's 16 bytes
        const float4 yy = *reinterpret_cast<const float4 *>(ddu + it_ddu + k * 2 * LY::DDU_ROW);
        const float2 ysum = zg_add2(make_float2(yy.x, yy.y), make_float2(yy.z, yy.w));
        const float2 u2 = pt_unpack2<T>(*reinterpret_cast<const uint32_t *>(raw + it_raw + k * 128));
        float2 y = zg_fma2(Dv, u2, ysum);
        if (has_z) y = zg_mul2(y, pt_silu2(pt_unpack2<T>(*reinterpret_cast<const uint32_t *>(raw + 2 * TILE + it_raw + k * 128))));
        uint32_t *dst = reinterpret_cast<uint32_t *>(gout + k * out_item);
        if (out_acc) {      // out = round(out + round(y)): the eager sum of two I/O-dtype tensors (mamba_simple.py:337)
            const float2 prev = pt_unpack2<T>(*dst), yr = pt_unpack2<T>(pt_pack2<T>(y.x, y.y));
            y = zg_add2(prev, yr);
        }
        *dst = pt_pack2<T>(y.x, y.y);
    };

    // ---- the pipeline ------------------------------------------------------------------------------------------------
    const unsigned char *ddu_j = ddu + (lane >> 1) * 16;
    const float *bq = bcf + 4 * part;
    unsigned char *ypart = ddu + (lane >> 1) * 16 + part * 8;
    zg_mbar_wait(&full[0], 0);       // stage 0: pre only
#pragma unroll
    for (int k = 0; k < NITEM; ++k) pre_item(k, smem);
    bc_convert(smem);
    __syncwarp();
    int slot = 0, nslot = 1;
    uint32_t npar = 0;                                             // phase parity of the next stage's slot
    for (int s = 0; s < nstages; ++s) {
        int sstep = -1;
        if (sync_every > 0 && --sync_left == 0) { sync_left = sync_every; sstep = sync_step; }
        wp2_main_stage<LY::DDU_ROW>(ddu_j, bq, ypart, h2, Al2p, sstep, cta_warps * 32);
        if constexpr (CKPT) {       // recompute seeds of the backward: state after every 8 steps, (batch, n_ckpt, dim, dstate)
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                float4 *dst = reinterpret_cast<float4 *>(p.ckpt + (((int64_t)b * (L >> 3) + s) * E + e + c) * 16 + 8 * part);
                dst[0] = make_float4(h2[c][0].x, h2[c][0].y, h2[c][1].x, h2[c][1].y);
                dst[1] = make_float4(h2[c][2].x, h2[c][2].y, h2[c][3].x, h2[c][3].y);
            }
        }
        const unsigned char *raw = smem + slot * LY::RAW;
        __syncwarp();               // partial y of the stage complete; B/C tile free
        if (s + 1 < nstages) {      // post(s) interleaved with pre(s + 1): independent MUFU chains
            const unsigned char *rawn = smem + nslot * LY::RAW;
            zg_mbar_wait(&full[nslot], npar);
#pragma unroll
            for (int k = 0; k < NITEM; ++k) { post_item(k, raw); pre_item(k, rawn); }
            bc_convert(rawn);
        } else {
#pragma unroll
            for (int k = 0; k < NITEM; ++k) post_item(k, raw);
        }
        gout += out_stage;
        __syncwarp();               // raw slot of stage s free; pairs and B/C of stage s + 1 complete
        issue_stage(slot);
        slot = nslot;
        if (++nslot == NSTAGE) { nslot = 0; npar ^= 1; }
    }
    if (p.last_state) {
#pragma unroll
        for (int c = 0; c < 2; ++c) {
            float4 *dst = reinterpret_cast<float4 *>(p.last_state + ((int64_t)b * E + e + c) * 16 + 8 * part);
            dst[0] = make_float4(h2[c][0].x, h2[c][0].y, h2[c][1].x, h2[c][1].y);
            dst[1] = make_float4(h2[c][2].x, h2[c][2].y, h2[c][3].x, h2[c][3].y);
        }
    }
}

template <typename T, bool CKPT, bool PLAIN, bool TMA>
__global__ void __launch_bounds__(32 * WP2_MAX_WARPS, 2) scan_fwd_wp2_kernel(const zg_scan_params p, const __grid_constant__ PtMaps maps) {
    extern __shared__ __align__(1024) unsigned char smem_all[];
    const int lane = threadIdx.x & 31;
    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);   // warp-uniform for the compiler
    const int per_group = p.dim / p.ngroups;
    const int units_per_group = per_group / WP2_CH;
    const int units = units_per_group * p.ngroups;                 // 32-channel units of a batch row
    const int wu = blockIdx.x * (int)(blockDim.x >> 5) + warp;     // warps are independent: any number of them per CTA
    if (wu >= units * p.batch) return;
    const int unit = wu % units;
    wp2_body<T, CKPT, PLAIN, TMA>(p, maps, smem_all + warp * Wp2Layout::WARP_BYTES, lane, wu / units, unit / units_per_group, unit * WP2_CH);
}

// CTA shape: see wp_pick_shape.  Half the warps of the one-channel-per-lane kernel: up to 18 per SM (112 registers) in two CTAs.
inline int wp2_pick_warps(long long units, int sms) {
    const int forced = pt_env_int("ZG_SCAN_WP_WARPS", 0);
    if (forced >= 1 && forced <= WP2_MAX_WARPS) return forced;
    if (units > 18LL * sms) return 3;                                        // several waves: six small CTAs per SM
    const long long per_sm = (units + sms - 1) / sms;                        // warps on the fullest SM
    const int ctas_per_sm = per_sm > 4 ? 2 : 1;
    return (int)((units + (long long)sms * ctas_per_sm - 1) / ((long long)sms * ctas_per_sm));
}

template <typename T, bool CKPT, bool PLAIN, bool TMA> int wp2_launch(const zg_scan_params &p, cudaStream_t stream) {
    using LY = Wp2Layout;
    PtMaps maps;
    memset(&maps, 0, sizeof(maps));
    if constexpr (TMA) {
        int rc = pt_make_map<T>(&maps.u, p.u, p.dim, p.seqlen, p.batch, p.u_sl, p.u_sb, WP2_CH, false);
        if (!rc) rc = pt_make_map<T>(&maps.d, p.delta, p.dim, p.seqlen, p.batch, p.delta_sl, p.delta_sb, WP2_CH, false);
        if (rc) return rc;
    }
    auto kern = scan_fwd_wp2_kernel<T, CKPT, PLAIN, TMA>;
    static bool attr_dev[64] = {};      // per instantiation and device
    static int sms_dev[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (!attr_dev[dev & 63]) {
        cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, WP2_MAX_WARPS * LY::WARP_BYTES);
        if (err != cudaSuccess) return zg_set_error("scan_fwd(wp2): cudaFuncSetAttribute(%d B smem): %s", WP2_MAX_WARPS * LY::WARP_BYTES, cudaGetErrorString(err));
        cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaDeviceGetAttribute(&sms_dev[dev & 63], cudaDevAttrMultiProcessorCount, dev);
        attr_dev[dev & 63] = true;
    }
    const long long units = (long long)(p.dim / WP2_CH) * p.batch;
    const int w = wp2_pick_warps(units, sms_dev[dev & 63] > 0 ? sms_dev[dev & 63] : 132);
    const long long nblk = (units + w - 1) / w;
    kern<<<(unsigned)nblk, 32 * w, w * LY::WARP_BYTES, stream>>>(p, maps);
    zg_count_launch();
    zg_note_scan_kernel(TMA ? "zg::scan_fwd_wp2_kernel (warp-private pipeline, 32 channels per warp, TMA tiles)" : "zg::scan_fwd_wp2_kernel (warp-private pipeline, 32 channels per warp, cp.async)");
    return zg_check_launch("scan_fwd(wp2)");
}

// mode: 3 = cp.async staging, 4 = TMA tiles for u / delta.  The caller (try_launch_scan_fwd_tma) has checked the shape class
// (dim / groups a multiple of 64, hence of 32).
template <typename T> int wp2_launch_variant(const zg_scan_params &p, cudaStream_t stream, int mode) {
    const bool plain = p.z && (p.flags & ZG_SCAN_DELTA_SOFTPLUS) && !(p.flags & (ZG_SCAN_OUT_REVERSE | ZG_SCAN_OUT_ACCUMULATE));
    if (mode == 4) {
        if (p.ckpt) return wp2_launch<T, true, false, true>(p, stream);
        return plain ? wp2_launch<T, false, true, true>(p, stream) : wp2_launch<T, false, false, true>(p, stream);
    }
    if (p.ckpt) return wp2_launch<T, true, false, false>(p, stream);
    return plain ? wp2_launch<T, false, true, false>(p, stream) : wp2_launch<T, false, false, false>(p, stream);
}

}  // namespace zg
