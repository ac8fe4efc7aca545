"""Worker for tests/test_gpu_cross_attention.py: 3 training steps of has_text ZigMa models, printing sha256 digests of
everything the steps produce.  Run twice in fresh processes, the digests must be equal.

    python tests/_xattn_det_worker.py [model ...]      (default: every model below)

Per model: fp32 parameters, 3 train_steps with FusedAdamWEMA, once plain and once under bf16 autocast (digests of the flat
parameters, both Adam moments, the EMA and the losses); bf16 parameters, 3 steps of forward + backward + plain SGD update
(FusedAdamWEMA keeps fp32 parameters; digests of every parameter gradient of the last step, the parameters and the losses).
One line per result: "DIGEST <model> <mode> <what> <sha256>"."""
import hashlib
import os
import sys

os.environ["CUBLAS_WORKSPACE_CONFIG"] = ":4096:8"       # before CUDA initialises: cuBLAS's deterministic workspace
import torch  # noqa: E402

torch.use_deterministic_algorithms(True)

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from zigma_b200 import ZigMa, create_transport  # noqa: E402
from zigma_b200.train import FlatParams, FusedAdamWEMA, train_step  # noqa: E402

MODELS = {   # name -> (config, latent shape, text tokens)
    "tiny_text": (dict(img_dim=8, patch_size=1, in_channels=4, embed_dim=64, depth=2, scan_type="zigzagN8", use_pe=0, drop_path_rate=0.0,
                       has_text=True, d_context=24), (4, 4, 8, 8), 7),
    # the reference's demo width (D 768, 77 CLIP tokens of width 768), 32 x 32 latents at patch 2: L = 256
    "demo_width": (dict(img_dim=32, patch_size=2, in_channels=4, embed_dim=768, depth=2, scan_type="zigzagN8", use_pe=2, drop_path_rate=0.0,
                        has_text=True, d_context=768), (2, 4, 32, 32), 77),
}


def digest(t):
    return hashlib.sha256(t.detach().contiguous().reshape(-1).view(torch.uint8).cpu().numpy().tobytes()).hexdigest()


def build(name, dtype):
    cfg, shape, ntok = MODELS[name]
    torch.manual_seed(0)
    m = ZigMa(device="cuda", dtype=dtype, **cfg)
    with torch.no_grad():                 # adaLN-zero init would leave the attention branch without gradient
        for p in m.parameters():
            if p.requires_grad and p.abs().sum() == 0:
                p.normal_(0, 0.02)
    m.eval()                              # drop_path off; gradients flow
    g = torch.Generator(device="cuda").manual_seed(1)
    x1 = torch.randn(shape, device="cuda", generator=g).to(dtype)
    y = torch.randn(shape[0], ntok, cfg["d_context"], device="cuda", generator=g).to(dtype)
    return m, x1, {"y": y}


def run(name):
    tr = create_transport()
    for mode, autocast in (("fp32", None), ("amp", torch.bfloat16)):
        m, x1, kw = build(name, torch.float32)
        flat = FlatParams(m)
        opt = FusedAdamWEMA(flat, lr=1e-3, weight_decay=0.01, ema_decay=0.99)
        losses = []
        for it in range(3):
            torch.manual_seed(10 + it)
            losses.append(train_step(m, tr, opt, None, x1, kw, autocast_dtype=autocast))
        torch.cuda.synchronize()
        for what, t in (("params", flat.flat), ("exp_avg", opt.exp_avg), ("exp_avg_sq", opt.exp_avg_sq), ("ema", opt.ema),
                        ("losses", torch.stack(losses))):
            print(f"DIGEST {name} {mode} {what} {digest(t)}", flush=True)
    m, x1, kw = build(name, torch.bfloat16)
    losses = []
    for it in range(3):
        torch.manual_seed(10 + it)
        m.zero_grad(set_to_none=True)
        loss = tr.training_losses(m, x1, kw)["loss"].float().mean()
        loss.backward()
        with torch.no_grad():
            for p in m.parameters():
                if p.grad is not None:
                    p.add_(p.grad, alpha=-1e-3)
        losses.append(loss.detach())
    torch.cuda.synchronize()
    for n, p in m.named_parameters():
        if p.grad is not None:
            print(f"DIGEST {name} bf16 grad:{n} {digest(p.grad)}", flush=True)
    print(f"DIGEST {name} bf16 params {digest(torch.cat([p.detach().reshape(-1) for p in m.parameters()]))}", flush=True)
    print(f"DIGEST {name} bf16 losses {digest(torch.stack(losses))}", flush=True)


if __name__ == "__main__":
    assert torch.are_deterministic_algorithms_enabled()
    for name in sys.argv[1:] or list(MODELS):
        run(name)
    print("XATTN_DET_WORKER_OK", flush=True)
