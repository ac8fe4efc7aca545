"""Worker for tests/test_gpu_drop_path.py: train-mode training steps (stochastic depth active, drop_path_rate 0.1) of small
ZigMa models with PyTorch's deterministic mode on, printing sha256 digests of everything the steps produce.  Run twice in
fresh processes, the digests must be equal.  (tests/_det_train_worker.py covers the same in eval mode.)

    python tests/_droppath_det_worker.py [model ...]

Per model: fp32 parameters, 3 train_steps with FusedAdamWEMA, once plain and once under bf16 autocast; bf16 parameters,
3 forward + backward passes.  One line per result: "DIGEST <model> <mode> <what> <sha256>"."""
import hashlib
import os
import sys

os.environ["CUBLAS_WORKSPACE_CONFIG"] = ":4096:8"       # before CUDA initialises: cuBLAS's deterministic workspace
import torch  # noqa: E402

torch.use_deterministic_algorithms(True)

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from zigma_b200 import ZigMa, create_transport  # noqa: E402
from zigma_b200.model_zigma import DropPath  # noqa: E402
from zigma_b200.train import FlatParams, FusedAdamWEMA, train_step  # noqa: E402

# depth 6: blocks 2..5 hold an active DropPath (rates 0.02 .. 0.1), as in the reference's default recipe
_TINY = dict(img_dim=8, patch_size=1, in_channels=4, embed_dim=64, depth=6, drop_path_rate=0.1)
MODELS = {
    "zigzagN8": (dict(_TINY, scan_type="zigzagN8", use_pe=0), (8, 4, 8, 8)),
    "v2": (dict(_TINY, scan_type="v2", use_pe=2), (8, 4, 8, 8)),
}


def digest(t):
    return hashlib.sha256(t.detach().contiguous().reshape(-1).view(torch.uint8).cpu().numpy().tobytes()).hexdigest()


def build(name, dtype):
    cfg, shape = MODELS[name]
    torch.manual_seed(0)
    m = ZigMa(device="cuda", dtype=dtype, **cfg)
    with torch.no_grad():                 # adaLN-zero init would leave every gradient but the head's zero
        for p in m.parameters():
            if p.requires_grad and p.abs().sum() == 0:
                p.normal_(0, 0.02)
    m.train()
    assert m._fused_tail_ok(torch.empty(1, 1, 64, device="cuda", dtype=dtype))
    assert sum(isinstance(b.drop_path, DropPath) for b in m.blocks) == 4
    g = torch.Generator(device="cuda").manual_seed(1)
    x1 = torch.randn(shape, device="cuda", generator=g).to(dtype)
    return m, x1


def run(name):
    tr = create_transport()
    for mode, autocast in (("fp32", None), ("amp", torch.bfloat16)):
        m, x1 = build(name, torch.float32)
        flat = FlatParams(m)
        opt = FusedAdamWEMA(flat, lr=1e-3, weight_decay=0.01, ema_decay=0.99)
        losses = []
        for it in range(3):
            torch.manual_seed(10 + it)
            losses.append(train_step(m, tr, opt, None, x1, {}, autocast_dtype=autocast))
        torch.cuda.synchronize()
        for what, t in (("params", flat.flat), ("exp_avg", opt.exp_avg), ("exp_avg_sq", opt.exp_avg_sq), ("ema", opt.ema),
                        ("losses", torch.stack(losses)), ("cuda_rng", torch.cuda.get_rng_state())):
            print(f"DIGEST {name} {mode} {what} {digest(t)}", flush=True)
    # bf16 parameters (FusedAdamWEMA keeps fp32 masters only): 3 forward + backward passes, each with its own draws
    m, x1 = build(name, torch.bfloat16)
    for it in range(3):
        m.zero_grad(set_to_none=True)
        torch.manual_seed(10 + it)
        loss = tr.training_losses(m, x1, {})["loss"].float().mean()
        loss.backward()
        print(f"DIGEST {name} bf16 loss{it} {digest(loss)}", flush=True)
    for n, p in m.named_parameters():
        if p.grad is not None:
            print(f"DIGEST {name} bf16 grad:{n} {digest(p.grad)}", flush=True)
    print(f"DIGEST {name} bf16 cuda_rng {digest(torch.cuda.get_rng_state())}", flush=True)


if __name__ == "__main__":
    assert torch.are_deterministic_algorithms_enabled()
    for name in sys.argv[1:] or list(MODELS):
        run(name)
    print("DROPPATH_DET_WORKER_OK", flush=True)
