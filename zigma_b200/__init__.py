"""zigma_b200 -- H100-native (sm_90a) implementation of the ZigMa denoiser hot path.

Public surface mirrors the reference (CompVis/zigma):
    ZigMa, Mamba, selective_scan_fn, mamba_inner_fn, mamba_inner_fn_no_out_proj, bimamba_inner_fn,
    causal_conv1d_fn, rms_norm_fn, layer_norm_fn, RMSNorm, zigzag_path, hilbert_path,
    reverse_permut_np, create_transport, Sampler
plus what sits around the path on an H100 node: train_step / FlatParams / GradSync / FusedAdamWEMA (zigma_b200.train),
load_reference_checkpoint / save_reference_checkpoint (zigma_b200.checkpoint), decode_latents / to_uint8_pixels (zigma_b200.handoff:
the VAE-decode hand-off after sampling).
All arithmetic on the path runs in libzigma_b200.so (include/zigma_b200.h); there is no CPU fallback.
"""
from .utils_zigzag import zigzag_path, hilbert_path, reverse_permut_np  # noqa: F401  (pure numpy, always importable)


def __getattr__(name):
    # torch-dependent symbols are imported lazily so the integer tables stay usable without CUDA
    import importlib
    table = {
        "ZigMa": "model_zigma", "Block": "model_zigma", "Mamba": "mamba_simple",
        "selective_scan_fn": "selective_scan_interface", "mamba_inner_fn": "selective_scan_interface",
        "mamba_inner_fn_no_out_proj": "selective_scan_interface", "bimamba_inner_fn": "selective_scan_interface",
        "causal_conv1d_fn": "causal_conv1d_interface", "rms_norm_fn": "layernorm", "layer_norm_fn": "layernorm",
        "RMSNorm": "layernorm", "ZigMaEngine": "engine", "create_transport": "transport", "Sampler": "transport",
        "mamba_inner_tok_fn": "selective_scan_interface", "block_tail_fn": "block_ops",
        "FlatParams": "train", "GradSync": "train", "FusedAdamWEMA": "train", "train_step": "train",
        "load_reference_checkpoint": "checkpoint", "save_reference_checkpoint": "checkpoint",
        "decode_latents": "handoff", "to_uint8_pixels": "handoff", "sample_and_decode": "handoff",
    }
    if name in table:
        return getattr(importlib.import_module("." + table[name], __name__), name)
    raise AttributeError(name)
