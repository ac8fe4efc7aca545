"""Worker for tests/test_gpu_deterministic.py: a few training steps of small ZigMa models with PyTorch's deterministic mode
on, printing sha256 digests of everything the steps produce.  Run twice in fresh processes, the digests must be equal.

    python tests/_det_train_worker.py [model ...]      (default: every model below)

Per model: fp32 parameters, 3 train_steps with FusedAdamWEMA, once plain and once under bf16 autocast (digests of the flat
parameters, both Adam moments, the EMA and the losses); bf16 parameters, one forward + backward (digest of every parameter
gradient).  One line per result: "DIGEST <model> <mode> <what> <sha256>"."""
import hashlib
import os
import sys

os.environ["CUBLAS_WORKSPACE_CONFIG"] = ":4096:8"       # before CUDA initialises: cuBLAS's deterministic workspace
import torch  # noqa: E402

torch.use_deterministic_algorithms(True)

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from zigma_b200 import ZigMa, create_transport  # noqa: E402
from zigma_b200.train import FlatParams, FusedAdamWEMA, train_step  # noqa: E402

_TINY = dict(img_dim=8, patch_size=1, in_channels=4, embed_dim=64, depth=2, use_pe=0, drop_path_rate=0.0)
MODELS = {   # name -> (config, latent shape, number of classes or 0)
    "zigzagN8": (dict(_TINY, scan_type="zigzagN8"), (4, 4, 8, 8), 0),
    "hilbertN8_layernorm": (dict(_TINY, scan_type="hilbertN8", rms_norm=False), (4, 4, 8, 8), 0),      # unfused add + LayerNorm
    "zigzagN8_checkpoint": (dict(_TINY, scan_type="zigzagN8", use_checkpoint=True), (4, 4, 8, 8), 0),  # unfused, checkpointed blocks
    "v2": (dict(_TINY, scan_type="v2", use_pe=2), (4, 4, 8, 8), 0),
    "zzvideo_sst": (dict(_TINY, patch_size=2, scan_type="zzvideo_sst", use_pe=2, video_frames=4, tpe=True), (2, 4, 4, 8, 8), 0),
    "class_cond": (dict(_TINY, patch_size=2, scan_type="zigzagN8", use_pe=2, num_classes=10), (4, 4, 8, 8), 10),
    "config2_width": (dict(img_dim=32, patch_size=1, in_channels=4, embed_dim=640, depth=2, scan_type="zigzagN8", use_pe=0, drop_path_rate=0.0),
                      (8, 4, 32, 32), 0),
}


def digest(t):
    return hashlib.sha256(t.detach().contiguous().reshape(-1).view(torch.uint8).cpu().numpy().tobytes()).hexdigest()


def build(name, dtype):
    cfg, shape, ncls = MODELS[name]
    torch.manual_seed(0)
    m = ZigMa(device="cuda", dtype=dtype, **cfg)
    with torch.no_grad():                 # adaLN-zero init would leave every gradient but the head's zero
        for p in m.parameters():
            if p.requires_grad and p.abs().sum() == 0:
                p.normal_(0, 0.02)
    m.eval()                              # drop_path off; gradients flow
    g = torch.Generator(device="cuda").manual_seed(1)
    x1 = torch.randn(shape, device="cuda", generator=g).to(dtype)
    y = torch.randint(0, ncls, (shape[0],), device="cuda", generator=g) if ncls else None
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
    torch.manual_seed(10)
    loss = tr.training_losses(m, x1, kw)["loss"].float().mean()
    loss.backward()
    for n, p in m.named_parameters():
        if p.grad is not None:
            print(f"DIGEST {name} bf16 grad:{n} {digest(p.grad)}", flush=True)
    print(f"DIGEST {name} bf16 loss {digest(loss)}", flush=True)


if __name__ == "__main__":
    assert torch.are_deterministic_algorithms_enabled()
    for name in sys.argv[1:] or list(MODELS):
        run(name)
    print("DET_WORKER_OK", flush=True)
