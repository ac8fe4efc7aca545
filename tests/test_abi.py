"""CPU: the C-ABI library builds, loads, exports every symbol include/zigma_b200.h declares, and the
ctypes Structures of zigma_b200/_lib.py have exactly the layout the C compiler gives the structs.
No compute call is made here (no GPU)."""
import ctypes
import os
import re
import subprocess
import tempfile

import pytest

from util import ROOT

HEADER = os.path.join(ROOT, "include", "zigma_b200.h")


def _declared():
    src = open(HEADER).read()
    return sorted(set(re.findall(r"\b(zg_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_entry_points():
    names = _declared()
    for n in ("zg_selective_scan_fwd", "zg_selective_scan_bwd", "zg_causal_conv1d_fwd", "zg_causal_conv1d_bwd",
              "zg_add_norm_fwd", "zg_add_norm_bwd", "zg_block_tail_fwd", "zg_block_tail_bwd", "zg_gemm_bf16_tn", "zg_gemm_kernel_choice",
              "zg_adamw_ema_step", "zg_last_error"):
        assert n in names


def test_library_exports_every_declared_symbol():
    import __graft_entry__
    __graft_entry__.build()
    from zigma_b200 import _lib
    assert os.path.exists(_lib.LIB_PATH)
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for n in _declared():
        assert hasattr(lib, n), f"{n} declared in include/zigma_b200.h but not exported"
    assert set(_lib.EXPORTS) == set(_declared())
    lib.zg_abi_version.restype = ctypes.c_int
    assert lib.zg_abi_version() >= 1


def test_ctypes_struct_layout_matches_c():
    from zigma_b200 import _lib
    structs = {"zg_scan_params": _lib.ScanParams, "zg_scan_bwd_params": _lib.ScanBwdParams,
               "zg_conv_params": _lib.ConvParams, "zg_conv_bwd_params": _lib.ConvBwdParams,
               "zg_norm_params": _lib.NormParams, "zg_norm_bwd_params": _lib.NormBwdParams,
               "zg_block_tail_params": _lib.BlockTailParams, "zg_block_tail_bwd_params": _lib.BlockTailBwdParams,
               "zg_gemm_params": _lib.GemmParams, "zg_adamw_params": _lib.AdamWParams}
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{HEADER}"', "int main(void) {"]
    for cname, st in structs.items():
        lines.append(f'printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, _ in st._fields_:
            lines.append(f'printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    lines.append("return 0; }")
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "l.c"), os.path.join(d, "l")
        open(src, "w").write("\n".join(lines))
        subprocess.check_call(["gcc", "-o", exe, src])
        out = subprocess.check_output([exe]).decode().split("\n")
    c_layout = dict(l.split() for l in out if l)
    for cname, st in structs.items():
        assert int(c_layout[cname]) == ctypes.sizeof(st), cname
        for fname, _ in st._fields_:
            assert int(c_layout[f"{cname}.{fname}"]) == getattr(st, fname).offset, f"{cname}.{fname}"


def test_ops_fail_loudly_without_cuda():
    """The product path has no CPU fallback: CPU tensors raise instead of silently computing."""
    import torch
    from zigma_b200 import selective_scan_fn, causal_conv1d_fn, rms_norm_fn
    if torch.cuda.is_available():
        pytest.skip("CPU-only behaviour")
    u = torch.randn(1, 4, 8)
    with pytest.raises(RuntimeError):
        selective_scan_fn(u, u, -torch.rand(4, 2), torch.randn(1, 2, 8), torch.randn(1, 2, 8))
    with pytest.raises(RuntimeError):
        causal_conv1d_fn(u, torch.randn(4, 3))
    with pytest.raises(RuntimeError):
        rms_norm_fn(torch.randn(2, 8), torch.ones(8), None)
    from zigma_b200.block_ops import block_tail_fn
    with pytest.raises(RuntimeError):
        block_tail_fn(torch.randn(1, 4, 8), None, None, torch.zeros(1, 8), torch.zeros(1, 8), torch.ones(8), None, None, 1e-5)


def test_scan_kernel_choice_shape_rule():
    """zg_scan_kernel_choice (the pure part of scan_auto_choice, scan_fwd.cuh): which hot-path forward-scan kernel a call gets on a
    132-SM H100.  The BASELINE workloads per GPU: config 2 (more than 36 units per SM: several waves), FacesHQ-1024 and both video
    layer shapes -> 32-channel warps, small batches and the training forward -> the CTA-wide kernel; one-wave batches in between
    -> mixed CTAs of wide + narrow warps."""
    from zigma_b200 import _lib
    ch = _lib.scan_kernel_choice
    assert ch(64, 1280) == (3, 0, 0)                       # zigzag8_b1 / sweep2_b1, bs 64
    assert ch(64, 1280, sms=148) == (5, 8, 2)              # (the same call on a device of 148 SMs: 8 wide + 2 narrow warps)
    assert ch(32, 1536) == (3, 0, 0)                       # faceshq1024, bs 32
    assert ch(16 * 16, 1536) == (3, 0, 0)                  # ucf101_sst spatial layers: 256 sequences
    assert ch(16 * 256, 1536) == (3, 0, 0)                 # ucf101_sst temporal layers: 4096 sequences
    assert ch(16, 1280) == (0, 0, 0) and ch(2, 128) == (0, 0, 0)
    assert ch(64, 1280, training_forward=True) == (0, 0, 0)
    mode, nd, ns = ch(32, 1280)
    assert (mode, nd, ns) == (5, 4, 2)
    for bs in range(1, 200):                               # whatever is picked is launchable: <= 10 warps, even narrow count, wide in fours
        mode, nd, ns = ch(bs, 1280)
        assert mode in (0, 3, 5)
        if mode == 5:
            assert nd in (4, 8) and ns % 2 == 0 and 0 <= ns and nd + ns <= 10
            units_per_sm = -(-bs * 80 // 132)
            assert 2 * (2 * nd + ns) >= units_per_sm       # two CTAs per SM hold the SM's share: one wave
