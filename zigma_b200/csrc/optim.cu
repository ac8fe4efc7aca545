// Fused AdamW + EMA step over one FLAT fp32 parameter buffer (sm_90a).
//
// Replaces, for the training loop around the denoiser (train_acc.py:442-448 of the reference):
//   opt.step()                      torch.optim.AdamW (lr, weight_decay; betas (0.9, 0.999), eps 1e-8 defaults, :213-215)
//   update_ema(ema_model, model)    one mul_ + one add_ per parameter tensor (utils/train_utils.py:104-115): ~660 launches
// by ONE pass: p, g, m, v, ema are read once and p, m, v, ema written once as 16-byte vectors -- 36 bytes per
// parameter, pure HBM streaming (31 M parameters -> 1.1 GB -> ~0.2 ms at the measured peak).  Same arithmetic and
// operation order as torch.optim.AdamW's single-tensor path (decoupled decay first, then the moment updates,
// denom = sqrt(v) / sqrt(bias_correction2) + eps, step = lr / bias_correction1), so the result matches it to fp32
// rounding.  An optional per-call gradient scale (loss scaling / the mean over data-parallel ranks / a clip
// coefficient) is applied to g on the fly; g itself is not modified.
#include "zg_common.cuh"

namespace zg {

__global__ void __launch_bounds__(256) adamw_ema_kernel(const zg_adamw_params p) {
    const int64_t n4 = p.n >> 2;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const float gs = p.grad_scale_ptr ? p.grad_scale * *p.grad_scale_ptr : p.grad_scale;
    const float decay = 1.f - p.lr * p.weight_decay;
    const float step = p.lr / p.bias_correction1;
    const float rsb2 = rsqrtf(p.bias_correction2);
    const float b1 = p.beta1, b2 = p.beta2, ob1 = 1.f - p.beta1, ob2 = 1.f - p.beta2;
    const float ed = p.ema_decay, oed = 1.f - p.ema_decay;
    auto upd = [&](float &w, float g, float &m, float &v, float &e) {
        g *= gs;
        w *= decay;
        m = fmaf(b1, m, ob1 * g);          // exp_avg.lerp_(grad, 1 - beta1)
        v = fmaf(b2, v, ob2 * g * g);      // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
        const float denom = sqrtf(v) * rsb2 + p.eps;
        w -= step * (m / denom);
        e = fmaf(ed, e, oed * w);          // ema.mul_(decay).add_(param, alpha=1 - decay)
    };
    float4 *P = reinterpret_cast<float4 *>(p.param), *M = reinterpret_cast<float4 *>(p.exp_avg), *V = reinterpret_cast<float4 *>(p.exp_avg_sq);
    float4 *Em = reinterpret_cast<float4 *>(p.ema);
    const float4 *G = reinterpret_cast<const float4 *>(p.grad);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        float4 w = P[i], g = G[i], m = M[i], v = V[i];
        float4 e = Em ? Em[i] : make_float4(0.f, 0.f, 0.f, 0.f);
        upd(w.x, g.x, m.x, v.x, e.x); upd(w.y, g.y, m.y, v.y, e.y); upd(w.z, g.z, m.z, v.z, e.z); upd(w.w, g.w, m.w, v.w, e.w);
        P[i] = w; M[i] = m; V[i] = v;
        if (Em) Em[i] = e;
    }
    // tail (n % 4 elements)
    const int64_t t = (n4 << 2) + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < p.n) {
        float e = p.ema ? p.ema[t] : 0.f;
        upd(p.param[t], p.grad[t], p.exp_avg[t], p.exp_avg_sq[t], e);
        if (p.ema) p.ema[t] = e;
    }
}

}  // namespace zg

extern "C" int zg_adamw_ema_step(const zg_adamw_params *pp, void *stream) {
    ZG_REQUIRE(pp != nullptr, "adamw_ema_step: null params");
    const zg_adamw_params &p = *pp;
    ZG_REQUIRE(p.param && p.grad && p.exp_avg && p.exp_avg_sq, "adamw_ema_step: null tensor pointer");
    ZG_REQUIRE(p.n >= 0, "adamw_ema_step: negative size");
    const uintptr_t al = reinterpret_cast<uintptr_t>(p.param) | reinterpret_cast<uintptr_t>(p.grad) | reinterpret_cast<uintptr_t>(p.exp_avg) |
                         reinterpret_cast<uintptr_t>(p.exp_avg_sq) | reinterpret_cast<uintptr_t>(p.ema);
    ZG_REQUIRE(al % 16 == 0, "adamw_ema_step: buffers must be 16-byte aligned");
    ZG_REQUIRE(p.bias_correction1 > 0.f && p.bias_correction2 > 0.f, "adamw_ema_step: bias corrections must be positive (step >= 1)");
    if (p.n == 0) return 0;
    const int64_t n4 = (p.n + 3) >> 2;
    int64_t blocks = (n4 + 255) / 256;
    if (blocks > 132 * 8) blocks = 132 * 8;          // grid-stride: 8 CTAs of 256 threads per SM
    zg::adamw_ema_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(p);
    zg_count_launch();
    return zg_check_launch("adamw_ema_step");
}
