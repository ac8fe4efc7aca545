// Selective-scan forward, warp-private pipeline (round 2, second half): the arithmetic of scan_fwd_tma_kernel with every
// warp running its own staging ring -- no block barrier anywhere in the stage loop.
//
// Why (profile of scan_fwd_tma_kernel on the GPU it was first tuned on): the kernel is bounded by the MUFU pipe (16 exp2 + 4 per
// (b, e, l)), yet that pipe is busy only 76 % of the time.  10 % of the stall samples sit on the instruction after the two
// BAR.SYNC of a stage, and only 6.2 of the 8.65 resident warps per sub-partition are alive on average: the four warps of a CTA
// live on four different sub-partitions, each of which schedules oldest-first, so a warp that is favoured on its own
// sub-partition keeps waiting for a sibling that is starved on another one, the CTAs drift apart, and the last CTAs of an SM
// run the tail with too few warps to keep the pipe fed.  Here a warp owns 16 channels x 16 states of one batch row end to end
// (same thread mapping inside the recurrence: two threads per channel, eight states each), stages its own u / delta / z / B|C
// rows (8 steps per stage, 3-deep ring, one mbarrier per slot), converts its own copy of the B|C rows and orders its phases
// with __syncwarp only.  Price: the 64-byte B|C rows are fetched (from L2) and converted once per warp instead of once per
// CTA, global rows are touched in 32-byte pieces (one sector) instead of 128-byte lines.
// Results are bit-identical to scan_fwd_tma_kernel (same operations in the same order per channel).
//
// Staging, two variants behind one template flag: TMA = u and delta as cp.async.bulk.tensor.3d tiles (16 channels x 8 steps,
// dense 32-byte rows) issued by lane 0, or every 16-byte chunk by cp.async from the lane that owns it (no elected-lane code:
// the UTMALDG sequence costs the whole warp ~45 issue slots per stage, the copies 2 per lane).  z rows (gathered through
// z_rowmap or not) and the B|C rows are always 16-byte cp.async chunks.
// Semantics: selective_scan_fwd_kernel.cuh:153-171, :216-261, :280-298 (see scan_fwd_tma.cuh).
#pragma once
#include "scan_fwd_tma.cuh"
#include <algorithm>

namespace zg {

#ifndef ZG_SCAN_WP_SYNC_DEFAULT
#define ZG_SCAN_WP_SYNC_DEFAULT 0     // stages between two fairness barriers of a CTA (0: none -- measured: every setting loses, see wp_pick_shape)
#endif
#ifndef ZG_SCAN_WP_NPOLY_DEFAULT
#define ZG_SCAN_WP_NPOLY_DEFAULT 0
#endif
constexpr int WP_CH = 16;             // channels per warp
constexpr int WP_MAX_WARPS = 18;      // independent warps per CTA: chosen per launch (wp_pick_shape), at most this many

struct WpLayout {                     // per warp
    static constexpr int NSTAGE = 3;
    static constexpr int TILE = PT_TL * WP_CH * 2;                // 8 steps x 32 B
    static constexpr int RAW = 3 * TILE + PT_TL * 64;             // u | delta | z | B|C rows (64 B each)
    static constexpr int DDU_ROW = WP_CH * 8;                     // (delta', delta' u) fp32 pairs of one step
    static constexpr int DDU_OFF = NSTAGE * RAW;
    static constexpr int BCF_OFF = DDU_OFF + PT_TL * DDU_ROW;     // fp32 [step][B0..15 C0..15]
    static constexpr int BAR_OFF = BCF_OFF + PT_TL * 32 * 4;
    static constexpr int WARP_BYTES = ((BAR_OFF + NSTAGE * 8 + 127) / 128) * 128;
};

// The work of one warp: 16 channels [e0, e0 + 16) of group g of batch row b, all seqlen steps.  `smem`: the warp's WpLayout bytes.
// sync_every = K > 0: the cta_warps warps of the CTA that have work meet at a named barrier every K stages.  They exchange nothing --
// the barrier is a fairness throttle (see wp_pick_shape).  The warp arrives after step `sync_step` of the stage's recurrence loop: the
// callers hand out different steps (warp index % 8), so that the barrier equalises the warps' progress WITHOUT aligning their phases
// (a barrier at the stage boundary puts every warp into the MUFU-heavy recurrence at the same time: measured, every setting lost).
template <typename T, bool CKPT, bool PLAIN, bool TMA, int NPOLY>
__device__ __forceinline__ void wp_body(const zg_scan_params &p, const PtMaps &maps, unsigned char *smem, const int lane, const int b, const int g, const int e0,
                                        const int sync_every, const int cta_warps, const int sync_step = 0) {
    static_assert(sizeof(T) == 2, "16-bit I/O only");
    using LY = WpLayout;
    constexpr int NSTAGE = LY::NSTAGE, TL = PT_TL, TILE = LY::TILE, NPAIR = 4;
    unsigned char *ddu = smem + LY::DDU_OFF;
    float *bcf = reinterpret_cast<float *>(smem + LY::BCF_OFF);
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + LY::BAR_OFF);

    const int part = lane & 1;                                     // which 8 states of the channel
    const int E = p.dim, L = p.seqlen;
    const int e = e0 + (lane >> 1);                                // main phase: this thread's channel
    const bool has_z = PLAIN ? true : (p.z != nullptr);
    const bool softplus = PLAIN ? true : ((p.flags & ZG_SCAN_DELTA_SOFTPLUS) != 0);
    const int nstages = L / TL;
    int sync_left = sync_every;

    // ---- per-thread constants -----------------------------------------------------------------------------------
    zg_f2 Al2p[NPAIR], h2[NPAIR];
    bool a_pos = false;
#pragma unroll
    for (int k = 0; k < NPAIR; ++k) {
        const float2 a = *reinterpret_cast<const float2 *>(p.A + (int64_t)e * 16 + 8 * part + 2 * k);
        Al2p[k] = zg_mul2(a, zg_splat2(ZG_LOG2E));
        a_pos = a_pos || a.x > 0.f || a.y > 0.f;
        h2[k] = zg_splat2(0.f);
    }
    // NPOLY of the four state pairs take their exp2 from the FMA pipe (zg_ex2_poly2_neg: needs delta' A <= 0, i.e. a
    // softplus'ed delta and non-positive A; decided per warp)
    const bool use_poly = NPOLY > 0 && softplus && !__any_sync(0xffffffffu, a_pos);
    // pre / post items of a lane: channel pair lane % 8 at steps lane / 8 and lane / 8 + 4 of the stage (the same items in
    // both phases: post reads the partial y from the 16 bytes its own pre filled)
    const int pair = lane & 7, r0 = lane >> 3;
    const int it_raw = r0 * 32 + pair * 4;                         // byte offset in a 8 x 32 B tile; second item: + 128
    const int it_ddu = r0 * LY::DDU_ROW + pair * 16;               // second item: + 4 rows
    const float2 Dv = p.D ? *reinterpret_cast<const float2 *>(p.D + e0 + 2 * pair) : make_float2(0.f, 0.f);
    const float2 biasv = p.delta_bias ? *reinterpret_cast<const float2 *>(p.delta_bias + e0 + 2 * pair) : make_float2(0.f, 0.f);

    if (lane == 0) {        // full[s]: one cp.async arrival per lane and stage (+ the TMA issuer's expect_tx)
#pragma unroll
        for (int s = 0; s < NSTAGE; ++s) zg_mbar_init(&full[s], TMA ? 33 : 32);
        zg_mbar_fence_init();
    }
    __syncwarp();

    // ---- producer side of the lane --------------------------------------------------------------------------------
    // chunk `lane` of the B|C rows: step lane / 4, B or C, which 16 bytes
    const unsigned char *bc_src;
    uint32_t bc_step;
    {
        const int r = lane >> 2, w = (lane >> 1) & 1, j = lane & 1;
        const T *src = w ? reinterpret_cast<const T *>(p.C) + (int64_t)b * p.C_sb + (int64_t)g * p.C_sg + (int64_t)r * p.C_sl
                         : reinterpret_cast<const T *>(p.B) + (int64_t)b * p.B_sb + (int64_t)g * p.B_sg + (int64_t)r * p.B_sl;
        bc_src = reinterpret_cast<const unsigned char *>(src + j * 8);
        bc_step = (uint32_t)(w ? p.C_sl : p.B_sl) * (2u * TL);
    }
    // z chunk (lanes 0..15): row lane / 2 of the stage, 16-byte half lane % 2; the source row goes through z_rowmap when given.
    // batch element b of z: plain batch stride, or two-level (b / K, b % K) for the temporal video scan (zg_scan_params.z_batch_inner)
    const int zr = (lane >> 1) & 7, zj = lane & 1;
    const int64_t z_boff = p.z_batch_inner > 0 ? (int64_t)(b / p.z_batch_inner) * p.z_sb + (int64_t)(b % p.z_batch_inner) * p.z_sbi : (int64_t)b * p.z_sb;
    const unsigned char *zsrc = (has_z && lane < 16) ? reinterpret_cast<const unsigned char *>(reinterpret_cast<const T *>(p.z) + z_boff + e0 + zj * 8) : nullptr;
    const uint32_t z_sl2 = (uint32_t)p.z_sl * 2u;                  // byte offsets inside a batch element fit 32 bits (host check)
    const int32_t *zmap = p.z_rowmap;
    int zrow_next = (zsrc != nullptr) ? (zmap ? zmap[zr] : zr) : 0; // (permuted) source row of the NEXT stage to issue
    // cp.async staging of u (lanes 0..15) and delta (lanes 16..31): row (lane % 16) / 2, half lane % 2
    const unsigned char *ud_src = nullptr;
    uint32_t ud_step = 0;
    if constexpr (!TMA) {
        const int64_t sl = lane < 16 ? p.u_sl : p.delta_sl;
        const T *src = lane < 16 ? reinterpret_cast<const T *>(p.u) + (int64_t)b * p.u_sb : reinterpret_cast<const T *>(p.delta) + (int64_t)b * p.delta_sb;
        ud_src = reinterpret_cast<const unsigned char *>(src + (int64_t)zr * sl + e0 + zj * 8);
        ud_step = (uint32_t)sl * (2u * TL);
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
            zg_cp_async16(raw + lane * 16, ud_src);
            ud_src += ud_step;
        }
        if (zsrc != nullptr) {
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

    // ---- pre / post work of a lane's two items --------------------------------------------------------------------
    auto bc_convert = [&](const unsigned char *raw) {              // B | C rows -> fp32 [step][B0..15 C0..15]: chunk `lane`, 8 values
        const uint4 v = *reinterpret_cast<const uint4 *>(raw + 3 * TILE + lane * 16);
        const float2 a = pt_unpack2<T>(v.x), c = pt_unpack2<T>(v.y), d = pt_unpack2<T>(v.z), f = pt_unpack2<T>(v.w);
        float4 *dst = reinterpret_cast<float4 *>(bcf + lane * 8);      // (two-way bank conflict between lanes c and c + 4: two STS per stage, not worth a select)
        dst[0] = make_float4(a.x, a.y, c.x, c.y);
        dst[1] = make_float4(d.x, d.y, f.x, f.y);
    };
    auto pre_item = [&](int k, const unsigned char *raw) {         // bias, softplus, * u -> (delta', delta' u) pairs
        float2 dl = pt_unpack2<T>(*reinterpret_cast<const uint32_t *>(raw + TILE + it_raw + k * 128));
        dl = zg_add2(dl, biasv);
        if (softplus) dl = pt_softplus20_2(dl);
        const float2 du = zg_mul2(dl, pt_unpack2<T>(*reinterpret_cast<const uint32_t *>(raw + it_raw + k * 128)));
        *reinterpret_cast<float4 *>(ddu + it_ddu + k * 4 * LY::DDU_ROW) = make_float4(dl.x, du.x, dl.y, du.y);
    };
    // output rows: step l -> sequence position l, or seqlen - 1 - l (ZG_SCAN_OUT_REVERSE: the backward sweep of scan_type v2)
    const bool out_rev = PLAIN ? false : ((p.flags & ZG_SCAN_OUT_REVERSE) != 0), out_acc = PLAIN ? false : ((p.flags & ZG_SCAN_OUT_ACCUMULATE) != 0);
    const int64_t out_row = out_rev ? -p.out_sl : p.out_sl;
    T *gout = reinterpret_cast<T *>(p.out) + (int64_t)b * p.out_sb + (int64_t)(out_rev ? L - 1 - r0 : r0) * p.out_sl + e0 + 2 * pair;
    const int64_t out_item = 4 * out_row, out_stage = (int64_t)TL * out_row;
    auto post_item = [&](int k, const unsigned char *raw) {        // y = y_lo + y_hi + D u, SiLU(z) gate, store
        const float4 yy = *reinterpret_cast<const float4 *>(ddu + it_ddu + k * 4 * LY::DDU_ROW);   // (lo, hi) halves of 2 channels
        const float2 ysum = zg_add2(make_float2(yy.x, yy.z), make_float2(yy.y, yy.w));
        const float2 u2 = pt_unpack2<T>(*reinterpret_cast<const uint32_t *>(raw + it_raw + k * 128));
        float2 y = zg_fma2(Dv, u2, ysum);
        if (has_z) y = zg_mul2(y, pt_silu2(pt_unpack2<T>(*reinterpret_cast<const uint32_t *>(raw + 2 * TILE + it_raw + k * 128))));
        uint32_t *dst = reinterpret_cast<uint32_t *>(gout + (k ? out_item : 0));
        if (out_acc) {      // out = round(out + round(y)): the eager sum of two I/O-dtype tensors (mamba_simple.py:337)
            const float2 prev = pt_unpack2<T>(*dst), yr = pt_unpack2<T>(pt_pack2<T>(y.x, y.y));
            y = zg_add2(prev, yr);
        }
        *dst = pt_pack2<T>(y.x, y.y);
    };

    // ---- the pipeline ------------------------------------------------------------------------------------------------
    const unsigned char *ddu_c = ddu + (lane >> 1) * 8;
    const float *bcf_p = bcf + 8 * part;
    unsigned char *ypart = ddu + (lane >> 1) * 8 + part * 4;
    zg_mbar_wait(&full[0], 0);       // stage 0: pre only
    pre_item(0, smem);
    pre_item(1, smem);
    bc_convert(smem);
    __syncwarp();
    int slot = 0, nslot = 1;
    uint32_t npar = 0;                                             // phase parity of the next stage's slot
    for (int s = 0; s < nstages; ++s) {
        int sstep = -1;                                 // every warp of the CTA runs the same number of stages
        if (sync_every > 0 && --sync_left == 0) { sync_left = sync_every; sstep = sync_step; }
        if (NPOLY > 0 && use_poly) pt_main_stage<NPOLY, 2, LY::DDU_ROW>(ddu_c, bcf_p, ypart, LY::DDU_ROW, h2, Al2p, true, sstep, cta_warps * 32);
        else pt_main_stage<0, 2, LY::DDU_ROW>(ddu_c, bcf_p, ypart, LY::DDU_ROW, h2, Al2p, true, sstep, cta_warps * 32);
        if constexpr (CKPT) {       // recompute seeds of the backward: state after every 8 steps, (batch, n_ckpt, dim, dstate)
            float4 *dst = reinterpret_cast<float4 *>(p.ckpt + (((int64_t)b * (L >> 3) + s) * E + e) * 16 + 8 * part);
            dst[0] = make_float4(h2[0].x, h2[0].y, h2[1].x, h2[1].y);
            dst[1] = make_float4(h2[2].x, h2[2].y, h2[3].x, h2[3].y);
        }
        const unsigned char *raw = smem + slot * LY::RAW;
        __syncwarp();               // partial y of the stage complete; B/C tile free
        if (s + 1 < nstages) {      // post(s) interleaved with pre(s + 1): four independent MUFU chains per lane
            const unsigned char *rawn = smem + nslot * LY::RAW;
            zg_mbar_wait(&full[nslot], npar);
            post_item(0, raw); pre_item(0, rawn);
            post_item(1, raw); pre_item(1, rawn);
            bc_convert(rawn);
        } else {
            post_item(0, raw);
            post_item(1, raw);
        }
        gout += out_stage;
        __syncwarp();               // raw slot of stage s free; pairs and B/C of stage s + 1 complete
        issue_stage(slot);
        slot = nslot;
        if (++nslot == NSTAGE) { nslot = 0; npar ^= 1; }
    }
    if (p.last_state) {
        float4 *dst = reinterpret_cast<float4 *>(p.last_state + ((int64_t)b * E + e) * 16 + 8 * part);
        dst[0] = make_float4(h2[0].x, h2[0].y, h2[1].x, h2[1].y);
        dst[1] = make_float4(h2[2].x, h2[2].y, h2[3].x, h2[3].y);
    }
}

// (576 threads x 2 CTAs: the register cap that lets 36 warps live on an SM, 56 per thread)
template <typename T, bool CKPT, bool PLAIN, bool TMA, int NPOLY = 0>
__global__ void __launch_bounds__(32 * WP_MAX_WARPS, 2) scan_fwd_wp_kernel(const zg_scan_params p, const __grid_constant__ PtMaps maps, const int sync_every) {
    extern __shared__ __align__(1024) unsigned char smem_all[];
    const int lane = threadIdx.x & 31;
    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);   // warp-uniform for the compiler: barrier / tile addresses in uniform registers
    const int per_group = p.dim / p.ngroups;
    const int units_per_group = per_group / WP_CH;
    const int units = units_per_group * p.ngroups;                 // 16-channel units of a batch row
    const int wu = blockIdx.x * (int)(blockDim.x >> 5) + warp;     // warps are independent: any number of them per CTA
    if (wu >= units * p.batch) return;
    // warps of this CTA that have work (the last CTA may be short): the participants of the fairness barrier
    const int cta_warps = min((int)(blockDim.x >> 5), units * p.batch - (int)blockIdx.x * (int)(blockDim.x >> 5));
    const int unit = wu % units;
    wp_body<T, CKPT, PLAIN, TMA, NPOLY>(p, maps, smem_all + warp * WpLayout::WARP_BYTES, lane, wu / units, unit / units_per_group, unit * WP_CH, sync_every, cta_warps, warp & 7);
}

// CTA shape.  The warps exchange nothing, so the CTA size is free; what it decides is how the SM's warp schedulers treat the
// warps.  ncu of 4- / 5-warp CTAs: only 6.1 of the 8.75 resident warps per sub-partition are alive
// on average although every warp has the same work -- the schedulers favour the oldest warps, those finish at ~40 % of the
// kernel time, and the youngest ones run the tail with too few peers to keep the MUFU pipe busy (74 % over the whole kernel).
// When the whole problem fits one wave, the warps of an SM are therefore packed into ONE or TWO large CTAs whose warps meet at a
// barrier every `sync_every` stages: a warp that has run ahead sleeps and the laggards get the pipe, so the warps of a CTA finish
// together; with two CTAs per SM either of them alone (>= 4 warps per sub-partition) keeps the pipe busy while the other is
// starved, so unfairness BETWEEN the two costs nothing.  Problems of several waves keep small CTAs (finished CTAs are replaced).
struct WpShape { int warps, sync_every; };
inline WpShape wp_pick_shape(long long units, int sms) {
    const int forced = pt_env_int("ZG_SCAN_WP_WARPS", 0);
    const int sync_env = pt_env_int("ZG_SCAN_WP_SYNC", ZG_SCAN_WP_SYNC_DEFAULT);
    if (forced >= 1 && forced <= WP_MAX_WARPS) return {forced, sync_env};
    if (units > 36LL * sms) return {4, 0};                                   // several waves
    const long long per_sm = (units + sms - 1) / sms;                        // warps on the fullest SM
    const int ctas_per_sm = per_sm > WP_MAX_WARPS ? 2 : 1;
    const int w = (int)((units + (long long)sms * ctas_per_sm - 1) / ((long long)sms * ctas_per_sm));
    return {w, sync_env};
}

template <typename T, bool CKPT, bool PLAIN, bool TMA, int NPOLY = 0> int wp_launch(const zg_scan_params &p, cudaStream_t stream) {
    using LY = WpLayout;
    PtMaps maps;
    memset(&maps, 0, sizeof(maps));
    if constexpr (TMA) {
        int rc = pt_make_map<T>(&maps.u, p.u, p.dim, p.seqlen, p.batch, p.u_sl, p.u_sb, WP_CH, false);
        if (!rc) rc = pt_make_map<T>(&maps.d, p.delta, p.dim, p.seqlen, p.batch, p.delta_sl, p.delta_sb, WP_CH, false);
        if (rc) return rc;
    }
    auto kern = scan_fwd_wp_kernel<T, CKPT, PLAIN, TMA, NPOLY>;
    static bool attr_dev[64] = {};      // per instantiation and device
    static int sms_dev[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (!attr_dev[dev & 63]) {
        cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, WP_MAX_WARPS * LY::WARP_BYTES);
        if (err != cudaSuccess) return zg_set_error("scan_fwd(wp): cudaFuncSetAttribute(%d B smem): %s", WP_MAX_WARPS * LY::WARP_BYTES, cudaGetErrorString(err));
        cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaDeviceGetAttribute(&sms_dev[dev & 63], cudaDevAttrMultiProcessorCount, dev);
        attr_dev[dev & 63] = true;
    }
    const long long units = (long long)(p.dim / WP_CH) * p.batch;
    const WpShape sh = wp_pick_shape(units, sms_dev[dev & 63] > 0 ? sms_dev[dev & 63] : 132);
    const int w = sh.warps;
    const long long nblk = (units + w - 1) / w;
    kern<<<(unsigned)nblk, 32 * w, w * LY::WARP_BYTES, stream>>>(p, maps, sh.sync_every);
    zg_count_launch();
    zg_note_scan_kernel(TMA ? "zg::scan_fwd_wp_kernel (warp-private pipeline, 16 channels per warp, TMA tiles)" : "zg::scan_fwd_wp_kernel (warp-private pipeline, 16 channels per warp, cp.async)");
    return zg_check_launch("scan_fwd(wp)");
}

// mode: 1 = cp.async staging, 2 = TMA tiles for u / delta.  The caller (try_launch_scan_fwd_tma) has checked the shape class.
template <typename T> int wp_launch_variant(const zg_scan_params &p, cudaStream_t stream, int mode) {
    const bool plain = p.z && (p.flags & ZG_SCAN_DELTA_SOFTPLUS) && !(p.flags & (ZG_SCAN_OUT_REVERSE | ZG_SCAN_OUT_ACCUMULATE));
    if (mode == 2) {
        if (p.ckpt) return wp_launch<T, true, false, true>(p, stream);
        return plain ? wp_launch<T, false, true, true>(p, stream) : wp_launch<T, false, false, true>(p, stream);
    }
    if (p.ckpt) return wp_launch<T, true, false, false>(p, stream);
    // ZG_SCAN_WP_NPOLY=1: one of the four state pairs of a thread (25 % of the exponentials) on the FMA pipe; the model's call only
    if (plain && pt_env_int("ZG_SCAN_WP_NPOLY", ZG_SCAN_WP_NPOLY_DEFAULT) == 1) return wp_launch<T, false, true, false, 1>(p, stream);
    return plain ? wp_launch<T, false, true, false>(p, stream) : wp_launch<T, false, false, false>(p, stream);
}

}  // namespace zg
