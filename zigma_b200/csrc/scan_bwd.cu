// Selective-scan backward: C-ABI entry points (the kernels are in scan_bwd.cuh / scan_bwd_q4.cuh).
#include "scan_bwd.cuh"

// validation shared by both entry points
static int scan_bwd_validate(const zg_scan_bwd_params &q) {
    const zg_scan_params &p = q.fwd;
    ZG_REQUIRE(p.u && p.delta && p.A && p.B && p.C && q.dout && q.du && q.ddelta && q.dA && q.dB && q.dC, "selective_scan_bwd: null tensor pointer");
    ZG_REQUIRE(((p.flags & ZG_SCAN_VARIABLE_B) && (p.flags & ZG_SCAN_VARIABLE_C)) || p.ngroups == 1, "selective_scan_bwd: constant B / C come with one group");
    ZG_REQUIRE(!p.z || q.dz, "selective_scan_bwd: dz output required when z is given");
    ZG_REQUIRE(p.ckpt != nullptr && p.ckpt_every == zg::BWD_TS, "selective_scan_bwd: needs the forward checkpoints with ckpt_every == %d", zg::BWD_TS);
    ZG_REQUIRE(p.ngroups >= 1 && p.dim % p.ngroups == 0, "selective_scan_bwd: bad groups");
    ZG_REQUIRE(p.dtype == ZG_F32 || p.dtype == ZG_F16 || p.dtype == ZG_BF16, "selective_scan_bwd: bad dtype %d", p.dtype);
    return 0;
}

// partial-row regions of the deterministic backward, in the order of the kernel that runs the call (see the DET notes of
// scan_bwd_q4_kernel / scan_bwd_kernel)
static ZgDetLayout scan_bwd_det_layout(const zg_scan_bwd_params &q, void *ws) {
    const zg_scan_params &p = q.fwd;
    ZgDetLayout lay;
    lay.ws = static_cast<unsigned char *>(ws);
    if (p.batch <= 0 || p.seqlen <= 0 || p.ngroups < 1 || p.dim % p.ngroups != 0) return lay;
    const bool varB = p.flags & ZG_SCAN_VARIABLE_B, varC = p.flags & ZG_SCAN_VARIABLE_C;
    const bool q4 = zg::scan_bwd_q4_fits(q);
    const int64_t N = p.dstate, E = p.dim, Bt = p.batch;
    const int64_t tpg = (E / p.ngroups + 63) / 64;                       // channel tiles per group (64 channels per CTA in both kernels)
    const int64_t bc_rows = q4 ? tpg : 2 * tpg;                           // q4: one row per CTA; generic: one per warp
    const int64_t bc_n = Bt * p.ngroups * N * p.seqlen;
    lay.add(q.dA, Bt, E * N);
    lay.add(q.dB, varB ? bc_rows : Bt, varB ? bc_n : E * N);
    lay.add(q.dC, varC ? bc_rows : Bt, varC ? bc_n : E * N);
    lay.add(q.dD, Bt, E);
    lay.add(q.ddelta_bias, Bt, E);
    return lay;
}

extern "C" int zg_selective_scan_bwd(const zg_scan_bwd_params *qq, void *stream) {
    ZG_REQUIRE(qq != nullptr, "selective_scan_bwd: null params");
    const zg_scan_bwd_params &q = *qq;
    if (int rc = scan_bwd_validate(q)) return rc;
    if (q.fwd.batch == 0 || q.fwd.seqlen == 0) return 0;
    return scan_bwd_dispatch<false>(q, (cudaStream_t)stream);
}

extern "C" int64_t zg_selective_scan_bwd_det_workspace_bytes(const zg_scan_bwd_params *q) {
    return q ? scan_bwd_det_layout(*q, nullptr).bytes : 0;
}

extern "C" int zg_selective_scan_bwd_det(const zg_scan_bwd_params *qq, void *workspace, int64_t workspace_bytes, void *stream) {
    ZG_REQUIRE(qq != nullptr, "selective_scan_bwd_det: null params");
    if (int rc = scan_bwd_validate(*qq)) return rc;
    if (qq->fwd.batch == 0 || qq->fwd.seqlen == 0) return 0;
    const ZgDetLayout lay = scan_bwd_det_layout(*qq, workspace);
    ZG_REQUIRE_WORKSPACE(lay, workspace, workspace_bytes, "selective_scan_bwd_det");
    zg_scan_bwd_params q = *qq;                 // the kernel writes partial rows; the reduction adds them to the outputs
    q.dA = lay.reg[0].part;
    int i = 1;
    q.dB = lay.reg[i++].part;
    q.dC = lay.reg[i++].part;
    if (q.dD) q.dD = lay.reg[i++].part;
    if (q.ddelta_bias) q.ddelta_bias = lay.reg[i++].part;
    cudaStream_t s = (cudaStream_t)stream;
    if (int rc = zg_scan_bwd_launch_det(q, s)) return rc;
    return lay.reduce(s);
}
