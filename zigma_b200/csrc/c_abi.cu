// C-ABI entry points (include/zigma_b200.h): argument validation, dispatch, error string.
#include "zg_common.cuh"
#include "scan_fwd.cuh"
#include <atomic>
#include <string.h>

static thread_local char g_err[512] = "";
static std::atomic<uint64_t> g_launches{0};
static std::atomic<const char *> g_scan_kernel{""};

int zg_set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return 1;
}
void zg_note_scan_kernel(const char *name) { g_scan_kernel.store(name, std::memory_order_relaxed); }
void zg_count_launch(int n) { g_launches.fetch_add((uint64_t)n, std::memory_order_relaxed); }
int zg_check_launch(const char *what) {
    cudaError_t err = cudaPeekAtLastError();
    if (err != cudaSuccess) {
        cudaGetLastError();
        return zg_set_error("%s: kernel launch failed: %s", what, cudaGetErrorString(err));
    }
    return 0;
}

extern "C" {

int zg_abi_version(void) { return 5; }   // 5: deterministic backward entry points zg_*_bwd_det + workspace queries
// int zg_abi_version(void) { return 4; }   // 4: zg_block_tail_fwd_pe (positional embedding folded into the first tail)
// int zg_abi_version(void) { return 3; }   // 3: fused dt_proj prologue fields in zg_scan_params
// int zg_abi_version(void) { return 2; }   // 2: block-tail rstd + backward, AdamW+EMA step, (batch, n_ckpt, dim, dstate) checkpoints
const char *zg_last_error(void) { return g_err; }
uint64_t zg_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }
const char *zg_last_scan_kernel(void) { return g_scan_kernel.load(std::memory_order_relaxed); }
int zg_scan_kernel_choice(int64_t units16, int32_t sms, int32_t training_forward, int32_t *nd, int32_t *ns) {
    const zg::ScanChoice c = zg::scan_choice_for(units16, sms, training_forward != 0);
    if (nd) *nd = c.nd;
    if (ns) *ns = c.ns;
    return c.mode;
}

int zg_selective_scan_fwd(const zg_scan_params *pp, void *stream) {
    ZG_REQUIRE(pp != nullptr, "selective_scan_fwd: null params");
    const zg_scan_params &p = *pp;
    ZG_REQUIRE(p.dtype == ZG_F32 || p.dtype == ZG_F16 || p.dtype == ZG_BF16, "selective_scan_fwd: bad dtype %d", p.dtype);
    ZG_REQUIRE(p.batch >= 0 && p.dim > 0 && p.seqlen >= 0, "selective_scan_fwd: bad shape (%d, %d, %d)", p.batch, p.dim, p.seqlen);
    ZG_REQUIRE(p.dstate >= 1 && p.dstate <= 64, "selective_scan_fwd: dstate must be in [1, 64], got %d", p.dstate);
    ZG_REQUIRE(p.ngroups >= 1 && p.dim % p.ngroups == 0, "selective_scan_fwd: dim %d not divisible by groups %d", p.dim, p.ngroups);
    const bool fused_dt = p.dt_w != nullptr;
    ZG_REQUIRE(p.u && (p.delta || fused_dt) && p.A && p.B && p.C && p.out, "selective_scan_fwd: null tensor pointer");
    ZG_REQUIRE(!fused_dt || (p.dt_x && p.dt_rank > 0), "selective_scan_fwd: fused dt_proj prologue needs dt_x and dt_rank");
    const bool seq = !fused_dt && p.u_sl == 1 && p.delta_sl == 1 && p.out_sl == 1 && (!p.z || p.z_sl == 1);
    const bool dimc = p.u_sd == 1 && (fused_dt || p.delta_sd == 1) && p.out_sd == 1 && (!p.z || p.z_sd == 1);
    ZG_REQUIRE(seq || dimc, "selective_scan_fwd: u, delta, z, out must all have seq stride 1 or all have dim stride 1");
    // (seqlen == 1 or dim == 1 tensors satisfy both; prefer the reference layout)
    const bool use_seq = seq;
    const bool varB = p.flags & ZG_SCAN_VARIABLE_B, varC = p.flags & ZG_SCAN_VARIABLE_C;
    if (use_seq) {
        ZG_REQUIRE(!varB || p.B_sl == 1 || p.seqlen == 1, "selective_scan_fwd: B must have seq stride 1 for seq-contiguous activations");
        ZG_REQUIRE(!varC || p.C_sl == 1 || p.seqlen == 1, "selective_scan_fwd: C must have seq stride 1 for seq-contiguous activations");
        ZG_REQUIRE(p.z_rowmap == nullptr, "selective_scan_fwd: z_rowmap needs the dim-contiguous layout");
    } else {
        ZG_REQUIRE(!varB || p.B_sn == 1 || p.dstate == 1, "selective_scan_fwd: B must have dstate stride 1 for dim-contiguous activations");
        ZG_REQUIRE(!varC || p.C_sn == 1 || p.dstate == 1, "selective_scan_fwd: C must have dstate stride 1 for dim-contiguous activations");
    }
    ZG_REQUIRE(!p.ckpt || (p.ckpt_every > 0 && p.ckpt_every % 8 == 0), "selective_scan_fwd: ckpt_every must be a positive multiple of 8");
    if (p.batch == 0 || p.seqlen == 0) return 0;
    const bool constbc = !(varB && varC);
    cudaStream_t s = (cudaStream_t)stream;
    switch (p.dtype) {
        case ZG_F32: return zg::scan_fwd_f32(p, use_seq, constbc, s);
        case ZG_F16: return zg::scan_fwd_f16(p, use_seq, constbc, s);
        default: return zg::scan_fwd_bf16(p, use_seq, constbc, s);
    }
}

}  // extern "C"

