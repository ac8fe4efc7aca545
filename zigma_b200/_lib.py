"""ctypes binding of the C-ABI in include/zigma_b200.h (libzigma_b200.so, sm_90a).

There is NO fallback: if the shared library is missing or a call fails, a RuntimeError is raised
(the reference raises RuntimeError from TORCH_CHECK the same way, selective_scan.cpp:226-336).
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("ZIGMA_B200_LIB") or os.path.join(_HERE, "lib", "libzigma_b200.so")   # (override: kernel timing experiments)

ZG_F32, ZG_F16, ZG_BF16 = 0, 1, 2
SCAN_DELTA_SOFTPLUS, SCAN_VARIABLE_B, SCAN_VARIABLE_C, SCAN_OUT_REVERSE, SCAN_OUT_ACCUMULATE = 1, 2, 4, 8, 16
_DT = {torch.float32: ZG_F32, torch.float16: ZG_F16, torch.bfloat16: ZG_BF16}

vp, i64, i32, f32 = C.c_void_p, C.c_int64, C.c_int32, C.c_float


class ScanParams(C.Structure):
    _fields_ = ([(n, vp) for n in ("u", "delta", "z", "B", "C", "A", "D", "delta_bias", "z_rowmap", "out", "last_state", "ckpt")]
                + [(n, i64) for n in ("u_sb", "u_sd", "u_sl", "delta_sb", "delta_sd", "delta_sl", "z_sb", "z_sd", "z_sl",
                                      "out_sb", "out_sd", "out_sl", "B_sb", "B_sg", "B_sn", "B_sl", "C_sb", "C_sg", "C_sn", "C_sl")]
                + [(n, i32) for n in ("batch", "dim", "seqlen", "dstate", "ngroups", "dtype", "flags", "ckpt_every")]
                + [(n, vp) for n in ("dt_w", "dt_x")]
                + [(n, i64) for n in ("dt_w_ld", "dt_x_sb", "dt_x_sl")]
                + [(n, i32) for n in ("dt_rank", "z_batch_inner")]
                + [("z_sbi", i64)])


class ScanBwdParams(C.Structure):
    _fields_ = ([("fwd", ScanParams), ("dout", vp)]
                + [(n, i64) for n in ("dout_sb", "dout_sd", "dout_sl")]
                + [(n, vp) for n in ("du", "ddelta", "dz")]
                + [(n, i64) for n in ("du_sb", "du_sd", "du_sl", "ddelta_sb", "ddelta_sd", "ddelta_sl", "dz_sb", "dz_sd", "dz_sl")]
                + [(n, vp) for n in ("dA", "dD", "ddelta_bias", "dB", "dC")])


class ConvParams(C.Structure):
    _fields_ = ([(n, vp) for n in ("x", "weight", "bias", "x_rowmap", "out")]
                + [(n, i64) for n in ("x_sb", "x_sd", "x_sl", "out_sb", "out_sd", "out_sl")]
                + [(n, i32) for n in ("batch", "dim", "seqlen", "width", "dtype", "wdtype", "silu", "seg_len")])


class ConvBwdParams(C.Structure):
    _fields_ = ([("fwd", ConvParams), ("dout", vp)]
                + [(n, i64) for n in ("dout_sb", "dout_sd", "dout_sl")]
                + [("dx", vp)]
                + [(n, i64) for n in ("dx_sb", "dx_sd", "dx_sl")]
                + [(n, vp) for n in ("dweight", "dbias")])


class NormParams(C.Structure):
    _fields_ = ([(n, vp) for n in ("x", "residual", "weight", "bias", "y", "residual_out", "mean", "rstd")]
                + [(n, i64) for n in ("x_rs", "res_rs", "y_rs", "resout_rs")]
                + [(n, i32) for n in ("nrows", "ncols", "dtype", "res_dtype", "wdtype", "is_rms")]
                + [("eps", f32)])


class NormBwdParams(C.Structure):
    _fields_ = ([(n, vp) for n in ("dy", "dresidual", "x", "weight", "mean", "rstd", "dx", "dresidual_in", "dweight", "dbias")]
                + [(n, i64) for n in ("dy_rs", "dres_rs", "x_rs", "dx_rs", "dresin_rs")]
                + [(n, i32) for n in ("nrows", "ncols", "dtype", "res_dtype", "wdtype", "is_rms")])


class BlockTailParams(C.Structure):
    _fields_ = ([(n, vp) for n in ("x", "mix", "gate", "shift", "scale", "norm_w", "residual", "rowmap", "residual_out", "normed", "modded")]
                + [("mod_rs", i64)]
                + [(n, i32) for n in ("batch", "seqlen", "dim", "dtype", "final_layer")]
                + [("eps", f32), ("rstd", vp)])


class BlockTailBwdParams(C.Structure):
    _fields_ = ([(n, vp) for n in ("d_residual_out", "d_normed", "d_modded", "r", "rstd", "mix", "gate", "scale", "norm_w", "rowmap",
                                   "d_x", "d_mix", "d_residual_in", "dgate", "dshift", "dscale", "d_norm_w")]
                + [("mod_rs", i64)]
                + [(n, i32) for n in ("batch", "seqlen", "dim", "dtype", "nparts")])


class BlockTailDpParams(C.Structure):
    _fields_ = [("base", BlockTailParams), ("path_scale", vp)]


class BlockTailBwdDpParams(C.Structure):
    _fields_ = [("base", BlockTailBwdParams), ("path_scale", vp)]


class BlockTailRebuildParams(C.Structure):
    _fields_ = [("base", BlockTailParams), ("x_rstd", vp), ("x_norm_w", vp)]


class XattnParams(C.Structure):
    _fields_ = ([(n, vp) for n in ("q", "k", "v", "o", "lse")]
                + [(n, i64) for n in ("q_sb", "q_rs", "k_sb", "k_rs", "v_sb", "v_rs", "o_sb", "o_rs")]
                + [(n, i32) for n in ("batch", "L", "Lk", "heads", "dim", "dtype")])


class XattnBwdParams(C.Structure):
    _fields_ = ([("fwd", XattnParams)]
                + [(n, vp) for n in ("dout", "dq", "dk", "dv")]
                + [(n, i64) for n in ("dout_sb", "dout_rs", "dq_sb", "dq_rs", "dk_sb", "dk_rs", "dv_sb", "dv_rs")]
                + [("sms", i32)])


class TextPrologueParams(C.Structure):
    _fields_ = ([(n, vp) for n in ("x", "mix", "gate", "shift", "scale", "rowmap", "hidden", "q_in", "mean", "rstd")]
                + [("mod_rs", i64)]
                + [(n, i32) for n in ("batch", "seqlen", "dim", "dtype")]
                + [("eps", f32)])


class TextPrologueBwdParams(C.Structure):
    _fields_ = ([(n, vp) for n in ("d_hidden", "d_q", "hidden", "mix", "gate", "scale", "mean", "rstd", "rowmap", "d_x", "d_mix",
                                   "dgate", "dshift", "dscale")]
                + [("mod_rs", i64)]
                + [(n, i32) for n in ("batch", "seqlen", "dim", "dtype", "nparts")])


class GemmParams(C.Structure):
    _fields_ = ([(n, vp) for n in ("A", "B", "bias", "C", "out_rowmap")]
                + [(n, i64) for n in ("lda", "ldb", "ldc")]
                + [(n, i32) for n in ("M", "N", "K", "rows_per_batch")])


class AdamWParams(C.Structure):
    _fields_ = ([(n, vp) for n in ("param", "exp_avg", "exp_avg_sq", "ema", "grad", "grad_scale_ptr")]
                + [("n", i64)]
                + [(n, f32) for n in ("lr", "beta1", "beta2", "eps", "weight_decay", "bias_correction1", "bias_correction2",
                                      "ema_decay", "grad_scale")])


EXPORTS = ["zg_abi_version", "zg_last_error", "zg_launch_count", "zg_last_scan_kernel", "zg_scan_kernel_choice", "zg_selective_scan_fwd", "zg_selective_scan_bwd",
           "zg_causal_conv1d_fwd", "zg_causal_conv1d_bwd", "zg_add_norm_fwd", "zg_add_norm_bwd",
           "zg_block_tail_fwd", "zg_block_tail_fwd_pe", "zg_block_tail_bwd", "zg_block_tail_fwd_dp", "zg_block_tail_bwd_dp",
           "zg_block_tail_fwd_rebuild",
           "zg_gemm_bf16_tn", "zg_adamw_ema_step", "zg_text_prologue_fwd", "zg_text_prologue_bwd"]
# deterministic backward twins (zg_<op>_det + zg_<op>_det_workspace_bytes) of these entry points
DET_OPS = ["zg_selective_scan_bwd", "zg_causal_conv1d_bwd", "zg_add_norm_bwd", "zg_block_tail_bwd", "zg_block_tail_bwd_dp",
           "zg_text_prologue_bwd"]
EXPORTS += [n + s for n in DET_OPS for s in ("_det", "_det_workspace_bytes")]
# cross-attention (always atomic-free, so no _det twin); the last two have signatures of their own
EXPORTS += ["zg_cross_attn_fwd", "zg_cross_attn_bwd", "zg_cross_attn_bwd_workspace_bytes"]
EXPORTS += ["zg_gemm_kernel_choice"]

_lib = None


def lib():
    """Loads libzigma_b200.so (built by ``__graft_entry__.build()`` / ``zigma_b200/csrc/build.sh``)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"zigma_b200: native library {LIB_PATH} not found -- build it with "
                f"`python -c 'import __graft_entry__ as g; g.build()'` (nvcc, sm_90a). There is no CPU/PyTorch fallback.")
        l = C.CDLL(LIB_PATH)
        l.zg_last_error.restype = C.c_char_p
        l.zg_launch_count.restype = C.c_uint64
        l.zg_last_scan_kernel.restype = C.c_char_p
        l.zg_last_scan_kernel.argtypes = []
        l.zg_scan_kernel_choice.restype = C.c_int
        l.zg_scan_kernel_choice.argtypes = [C.c_int64, C.c_int32, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
        for name in EXPORTS[5:]:
            if name.endswith("_det_workspace_bytes"):
                getattr(l, name).restype = C.c_int64
                getattr(l, name).argtypes = [C.c_void_p]
            elif name.endswith("_det"):
                getattr(l, name).restype = C.c_int
                getattr(l, name).argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
            else:
                getattr(l, name).restype = C.c_int
                getattr(l, name).argtypes = [C.c_void_p, C.c_void_p]
        l.zg_cross_attn_bwd.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
        l.zg_cross_attn_bwd_workspace_bytes.restype = C.c_int64
        l.zg_cross_attn_bwd_workspace_bytes.argtypes = [C.c_void_p]
        l.zg_gemm_kernel_choice.argtypes = [C.c_int32, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
        _lib = l
    return _lib


def launch_count():
    return int(lib().zg_launch_count())


def scan_kernel_choice(batch, dim, sms=132, training_forward=False):
    """(mode, wide warps, narrow warps) the shape rule picks for a hot-path forward-scan call (zg_scan_kernel_choice; host arithmetic)."""
    nd, ns = C.c_int32(0), C.c_int32(0)
    mode = lib().zg_scan_kernel_choice(int(batch) * (int(dim) // 16), int(sms), int(bool(training_forward)), C.byref(nd), C.byref(ns))
    return int(mode), int(nd.value), int(ns.value)


def gemm_kernel_choice(M, N):
    """(tile width, cluster size) of the zg::gemm_bf16_tn_kernel instantiation that zg_gemm_bf16_tn launches for an M x N output
    (zg_gemm_kernel_choice; host arithmetic, with the ZG_GEMM_BN / ZG_GEMM_CLUSTER overrides of the current environment)."""
    bn, cl = C.c_int32(0), C.c_int32(0)
    if lib().zg_gemm_kernel_choice(int(M), int(N), C.byref(bn), C.byref(cl)) != 0:
        raise RuntimeError(f"zg_gemm_kernel_choice: {lib().zg_last_error().decode()}")
    return int(bn.value), int(cl.value)


def last_scan_kernel():
    """Name of the kernel the most recent selective-scan forward call launched."""
    return lib().zg_last_scan_kernel().decode()


def call(name, params):
    """Invokes an entry point on torch's current CUDA stream; raises RuntimeError on failure."""
    l = lib()
    stream = torch.cuda.current_stream().cuda_stream
    rc = getattr(l, name)(C.byref(params), C.c_void_p(stream))
    if rc != 0:
        raise RuntimeError(f"{name}: {l.zg_last_error().decode()}")


def det_workspace_bytes(name, params):
    """Bytes of partials workspace the deterministic twin of backward entry point `name` needs for these params (host only)."""
    return int(getattr(lib(), name + "_det_workspace_bytes")(C.byref(params)))


def call_bwd(name, params):
    """Invokes backward entry point `name` like ``call``; while ``torch.are_deterministic_algorithms_enabled()`` its
    deterministic twin ``name + "_det"`` runs instead, with a partials workspace from torch's allocator on the current
    device (the same gradients up to summation order, bitwise reproducible run to run)."""
    if not torch.are_deterministic_algorithms_enabled():
        return call(name, params)
    l = lib()
    nbytes = det_workspace_bytes(name, params)
    ws = torch.empty((nbytes,), dtype=torch.uint8, device=torch.device("cuda", torch.cuda.current_device()))
    stream = torch.cuda.current_stream().cuda_stream
    rc = getattr(l, name + "_det")(C.byref(params), C.c_void_p(ws.data_ptr() if nbytes else None), C.c_int64(nbytes), C.c_void_p(stream))
    if rc != 0:
        raise RuntimeError(f"{name}_det: {l.zg_last_error().decode()}")


def dt(t):
    try:
        return _DT[t.dtype if isinstance(t, torch.Tensor) else t]
    except KeyError:
        raise RuntimeError(f"zigma_b200: unsupported dtype {t.dtype if isinstance(t, torch.Tensor) else t}")


def ptr(t):
    return None if t is None else t.data_ptr()


def require_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("zigma_b200: expected CUDA tensors (the kernels are sm_90a only; there is no CPU path)")
