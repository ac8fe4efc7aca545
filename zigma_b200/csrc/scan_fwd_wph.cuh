// Selective-scan forward, warp-private pipeline, MIXED warps: `nd` warps of a CTA own 32 channels (two per lane, wp2_body) and
// `ns` warps own 16 (one per lane, wp_body).
//
// Why: the two-channels-per-lane warp keeps the MUFU pipe of its sub-partition 85 % busy (against 76-79 % of the one-channel
// kernels), but its unit of work is twice as large, and at BASELINE config 2 the work does not
// divide: 81 920 channels / 592 sub-partitions = 8.65 units of 16 channels.  Whole 32-channel warps put 5 of them = 10 units on
// the fullest sub-partition (smsp__inst_executed max / avg = 1.16) and the kernel takes as long as before.  Four 32-channel warps
// plus one 16-channel warp per sub-partition are 9 units: the quantisation of the one-channel kernels with (mostly) the
// efficiency of the two-channel one.  A CTA of nd + ns = 8 + 2 warps covers 18 consecutive 16-channel units; two such CTAs per
// SM.  Which sub-partition a warp lands on is the hardware's choice (observed: warps are dealt round-robin and the second CTA
// continues where the first stopped, so the 2 x 2 narrow warps -- the LAST warps of each CTA -- land on four different
// sub-partitions).  Per channel the operations and their order are those of scan_fwd_tma_kernel: results are bit-identical.
#pragma once
#include "scan_fwd_wp2.cuh"

namespace zg {

constexpr int WPH_MAX_WARPS = 10;     // 320 threads x 2 CTAs per SM: 102 registers per thread

template <typename T, bool PLAIN>
__global__ void __launch_bounds__(32 * WPH_MAX_WARPS, 2) scan_fwd_wph_kernel(const zg_scan_params p, const int nd, const int ns) {
    extern __shared__ __align__(1024) unsigned char smem_all[];
    const int lane = threadIdx.x & 31;
    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);   // warp-uniform for the compiler
    const int row_units = p.dim / WP_CH;                           // 16-channel units of a batch row (even; so is every group's count)
    const int group_units = row_units / p.ngroups;
    const long long total = (long long)row_units * p.batch;
    const long long first = (long long)blockIdx.x * (2 * nd + ns);  // the CTA's first unit (even: a 32-channel pair never straddles a row or a group)
    if (warp < nd) {
        const long long u = first + 2 * warp;
        if (u >= total) return;
        const int unit = (int)(u % row_units);
        wp2_body<T, PLAIN>(p, smem_all + warp * Wp2Layout::WARP_BYTES, lane, (int)(u / row_units), unit / group_units, unit * WP_CH);
    } else {
        const long long u = first + 2 * nd + (warp - nd);
        if (u >= total) return;
        const int unit = (int)(u % row_units);
        wp_body<T, PLAIN>(p, smem_all + nd * Wp2Layout::WARP_BYTES + (warp - nd) * WpLayout::WARP_BYTES, lane, (int)(u / row_units),
                          unit / group_units, unit * WP_CH);
    }
}

template <typename T, bool PLAIN> int wph_launch(const zg_scan_params &p, cudaStream_t stream, int nd, int ns) {
    auto kern = scan_fwd_wph_kernel<T, PLAIN>;
    static bool attr_dev[64] = {};      // per instantiation and device
    int dev = 0;
    cudaGetDevice(&dev);
    constexpr int MAX_SMEM = WPH_MAX_WARPS * Wp2Layout::WARP_BYTES;
    if (!attr_dev[dev & 63]) {
        cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_SMEM);
        if (err != cudaSuccess) return zg_set_error("scan_fwd(wph): cudaFuncSetAttribute(%d B smem): %s", MAX_SMEM, cudaGetErrorString(err));
        cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        attr_dev[dev & 63] = true;
    }
    const long long units = (long long)(p.dim / WP_CH) * p.batch;
    const int per_cta = 2 * nd + ns;
    const long long nblk = (units + per_cta - 1) / per_cta;
    kern<<<(unsigned)nblk, 32 * (nd + ns), nd * Wp2Layout::WARP_BYTES + ns * WpLayout::WARP_BYTES, stream>>>(p, nd, ns);
    zg_count_launch();
    zg_note_scan_kernel("zg::scan_fwd_wph_kernel (warp-private pipeline, CTAs of 32- and 16-channel warps, cp.async)");
    return zg_check_launch("scan_fwd(wph)");
}

// mode 5.  nd wide + ns narrow warps per CTA: the caller's choice (scan_auto_choice), else ZG_SCAN_WPH_ND / ZG_SCAN_WPH_NS
// (default 8 + 2).  The caller keeps checkpoint calls on the CTA-wide kernel.
template <typename T> int wph_launch_variant(const zg_scan_params &p, cudaStream_t stream, int nd, int ns) {
    if (nd <= 0) { nd = pt_env_int("ZG_SCAN_WPH_ND", 8); ns = pt_env_int("ZG_SCAN_WPH_NS", 2); }
    if (nd < 0 || ns < 0 || nd + ns < 1 || nd + ns > WPH_MAX_WARPS || (ns & 1)) { nd = 8; ns = 2; }     // (an even number of narrow warps: a CTA starts at an even unit)
    const bool plain = p.z && (p.flags & ZG_SCAN_DELTA_SOFTPLUS) && !(p.flags & (ZG_SCAN_OUT_REVERSE | ZG_SCAN_OUT_ACCUMULATE));
    return plain ? wph_launch<T, true>(p, stream, nd, ns) : wph_launch<T, false>(p, stream, nd, ns);
}

}  // namespace zg
