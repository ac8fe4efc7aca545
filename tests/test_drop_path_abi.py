"""CPU: the drop-path block-tail entry points (zg_block_tail_fwd_dp, zg_block_tail_bwd_dp and its _det twin) -- ctypes layout,
exports, the argument checks on empty batches (nothing can launch), the deterministic workspace size, a SASS audit of the
built library, and the DropPath draw the fused training loop shares with DropPath.forward."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import pytest
import torch

from util import ROOT

HEADER = os.path.join(ROOT, "include", "zigma_b200.h")
FAKE = 1 << 20            # stands in for device pointers: the checks read addresses (alignment) only, never memory
NEW_FUNCS = ("zg_block_tail_fwd_dp", "zg_block_tail_bwd_dp", "zg_block_tail_bwd_dp_det", "zg_block_tail_bwd_dp_det_workspace_bytes")


def _built():
    import __graft_entry__
    __graft_entry__.build()
    from zigma_b200 import _lib
    return _lib


def _ptrs(obj, names, base=FAKE):
    for i, n in enumerate(names):
        setattr(obj, n, base * (i + 1))


def test_ctypes_layout_matches_c():
    from zigma_b200 import _lib
    structs = {"zg_block_tail_dp_params": _lib.BlockTailDpParams, "zg_block_tail_bwd_dp_params": _lib.BlockTailBwdDpParams}
    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{HEADER}"', "int main(void) {"]
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
        assert int(c_layout[cname]) == C.sizeof(st), cname
        for fname, _ in st._fields_:
            assert int(c_layout[f"{cname}.{fname}"]) == getattr(st, fname).offset, f"{cname}.{fname}"
    assert _lib.BlockTailDpParams.path_scale.offset == C.sizeof(_lib.BlockTailParams)
    assert _lib.BlockTailBwdDpParams.path_scale.offset == C.sizeof(_lib.BlockTailBwdParams)


def test_declared_and_exported():
    _lib = _built()
    declared = set(re.findall(r"\b(zg_[a-z0-9_]+)\s*\(", open(HEADER).read()))
    l = _lib.lib()
    for n in NEW_FUNCS:
        assert n in declared and n in _lib.EXPORTS and hasattr(l, n), n
    assert "zg_block_tail_bwd_dp" in _lib.DET_OPS
    assert _lib.EXPORTS.index("zg_block_tail_fwd_dp") >= 5 and _lib.EXPORTS.index("zg_block_tail_bwd_dp") >= 5
    assert l.zg_abi_version() == 5


def _fwd(_lib, dtype=None, dim=640):
    """Valid forward params of an EMPTY batch (batch 0): every check runs before the empty-batch return."""
    dtype = _lib.ZG_BF16 if dtype is None else dtype
    q = _lib.BlockTailDpParams()
    p = q.base
    _ptrs(p, ["x", "mix", "norm_w", "residual", "residual_out", "normed", "modded", "rowmap"])
    esz = 4 if dtype == _lib.ZG_F32 else 2
    p.shift, p.scale, p.gate = FAKE * 64, FAKE * 64 + dim * esz, FAKE * 64 + 2 * dim * esz
    p.mod_rs = 3 * dim
    p.batch, p.seqlen, p.dim, p.dtype, p.eps = 0, 16, dim, dtype, 1e-5
    q.path_scale = FAKE * 128
    return q


def _bwd(_lib, dtype=None, dim=640, nparts=1):
    dtype = _lib.ZG_BF16 if dtype is None else dtype
    q = _lib.BlockTailBwdDpParams()
    p = q.base
    _ptrs(p, ["d_residual_out", "d_normed", "d_modded", "r", "rstd", "mix", "norm_w", "rowmap", "d_x", "d_mix", "d_residual_in",
              "dgate", "dshift", "dscale", "d_norm_w"])
    esz = 4 if dtype == _lib.ZG_F32 else 2
    p.scale, p.gate = FAKE * 64 + dim * esz, FAKE * 64 + 2 * dim * esz
    p.mod_rs = 3 * dim
    p.batch, p.seqlen, p.dim, p.dtype, p.nparts = 0, 16, dim, dtype, nparts
    q.path_scale = FAKE * 128
    return q


def _call(_lib, name, q):
    l = _lib.lib()
    if name.endswith("_det"):
        rc = getattr(l, name)(C.byref(q), C.c_void_p(None), C.c_int64(0), C.c_void_p(None))
    else:
        rc = getattr(l, name)(C.byref(q), C.c_void_p(None))
    return rc, l.zg_last_error().decode()


def test_forward_accepts_and_rejects_on_empty_batches():
    _lib = _built()
    for dt in (_lib.ZG_F32, _lib.ZG_F16, _lib.ZG_BF16):
        for dim in (36, 368, 640, 1024):
            rc, err = _call(_lib, "zg_block_tail_fwd_dp", _fwd(_lib, dt, dim))
            assert rc == 0, (dt, dim, err)

    def rejected(what, **kw):
        q = _fwd(_lib)
        for k, v in kw.items():
            setattr(q if k == "path_scale" else q.base, k, v)
        rc, err = _call(_lib, "zg_block_tail_fwd_dp", q)
        assert rc != 0, what
        return err

    assert "path_scale" in rejected("null path_scale", path_scale=None)
    assert "residual" in rejected("no residual", residual=None)
    assert "mix" in rejected("no mix", mix=None)
    assert "final_layer" in rejected("final layer", final_layer=1)
    q = _fwd(_lib, dim=1028)
    assert _call(_lib, "zg_block_tail_fwd_dp", q)[0] != 0, "dim 1028"
    assert "1024" in rejected("dim above 1024", dim=1536)
    # what the plain entry point rejects
    assert "aligned" in rejected("gate 2 bytes off", gate=FAKE * 64 + 2 * 640 * 2 + 2)
    assert "multiple of 4" in rejected("dim 38", dim=38)
    assert "16-byte" in rejected("x misaligned", x=FAKE + 8)
    assert "mix needs gate" in rejected("mix without gate", gate=None)
    assert "aligned" in rejected("path_scale misaligned", path_scale=FAKE * 128 + 1)
    q = _fwd(_lib, _lib.ZG_F32)
    q.path_scale = FAKE * 128 + 2                 # fp32 multipliers need 4-byte alignment
    assert _call(_lib, "zg_block_tail_fwd_dp", q)[0] != 0


@pytest.mark.parametrize("name", ["zg_block_tail_bwd_dp", "zg_block_tail_bwd_dp_det"])
def test_backward_accepts_and_rejects_on_empty_batches(name):
    _lib = _built()
    for dt in (_lib.ZG_F32, _lib.ZG_F16, _lib.ZG_BF16):
        for dim in (36, 368, 640, 768, 1024):
            rc, err = _call(_lib, name, _bwd(_lib, dt, dim))
            assert rc == 0, (name, dt, dim, err)

    def rejected(what, **kw):
        q = _bwd(_lib)
        for k, v in kw.items():
            setattr(q if k == "path_scale" else q.base, k, v)
        rc, err = _call(_lib, name, q)
        assert rc != 0, what
        return err

    assert "path_scale" in rejected("null path_scale", path_scale=None)
    assert "mix" in rejected("first block (no mix, gate, d_mix)", mix=None, gate=None, d_mix=None, dgate=None)
    assert "1024" in rejected("dim above 1024", dim=1028)
    assert "aligned" in rejected("gate 2 bytes off", gate=FAKE * 64 + 2 * 640 * 2 + 2)
    assert "go together" in rejected("mix without d_mix", d_mix=None)
    assert "nparts" in rejected("nparts 0", nparts=0)
    assert "aligned" in rejected("path_scale misaligned", path_scale=FAKE * 128 + 1)


def test_dp_det_workspace_bytes_equal_the_plain_query():
    _lib = _built()
    for B in (1, 3, 16, 64):
        for L in (1, 37, 1024):
            for D in (36, 640, 1024):
                for nparts in (max(1, (B + 3) // 4), 256):
                    for first_absent in (False, True):
                        q = _bwd(_lib, dim=D, nparts=nparts)
                        q.base.batch, q.base.seqlen = B, L
                        if first_absent:
                            q.base.dshift = None
                        plain = _lib.det_workspace_bytes("zg_block_tail_bwd", q.base)
                        assert _lib.det_workspace_bytes("zg_block_tail_bwd_dp", q) == plain, (B, L, D, nparts)
                        assert plain > 0


def test_sass_drop_path_instantiations():
    """6 forward (T x Q 1/2) and 24 backward (T x MAXQ 4/5/6/8 x DET) instantiations; no floating-point atomic or reduction
    in the DET ones (the pattern of test_deterministic_abi.py)."""
    from test_deterministic_abi import FLOAT_ATOMIC, _tool
    cuobjdump, filt = _tool("cuobjdump"), _tool("cu++filt")
    if cuobjdump is None or filt is None:
        pytest.skip("cuobjdump / cu++filt not available")
    _lib = _built()
    sass = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    funcs, cur = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur is not None:
            funcs[cur].append(line)
    names = list(funcs)
    demangled = subprocess.run([filt], input="\n".join(names), check=True, capture_output=True, text=True).stdout.splitlines()
    fwd, bwd, det = set(), set(), 0
    for mangled, dem in zip(names, demangled):
        m = re.search(r"zg::(block_tail_dp_(?:fwd|bwd)_kernel)<(.*)>\(", dem)
        if m is None:
            continue
        args = tuple({"(bool)1": "true", "(bool)0": "false"}.get(a.strip(), a.strip()) for a in m.group(2).split(","))
        args = tuple(re.sub(r"^\((?:int|unsigned int)\)", "", a) for a in args)
        if m.group(1) == "block_tail_dp_fwd_kernel":
            fwd.add(args)
        else:
            bwd.add(args)
            if args[-1] == "true":
                det += 1
                bad = [l.strip() for l in funcs[mangled] if FLOAT_ATOMIC.search(l)]
                assert not bad, f"{dem}: {bad[:3]}"
    T = ("float", "__half", "__nv_bfloat16")
    assert fwd == {(t, q) for t in T for q in ("1", "2")}
    assert bwd == {(t, q, d) for t in T for q in ("4", "5", "6", "8") for d in ("false", "true")}
    assert det == 12


def test_drop_path_draw_equals_forward_mask():
    """DropPath.draw (what the fused training loop applies) is the mask DropPath.forward multiplies by, bit for bit, and
    leaves the generator where forward leaves it."""
    from zigma_b200.model_zigma import DropPath
    for dtype in (torch.float32, torch.bfloat16, torch.float16):
        for p in (0.5, 0.1, 0.002, 1.0):
            dp = DropPath(p).train()
            x = torch.randn(64, 3, 8).to(dtype)
            torch.manual_seed(123)
            out = dp(x)
            state = torch.get_rng_state()
            torch.manual_seed(123)
            mask = dp.draw(x)
            assert torch.equal(torch.get_rng_state(), state)
            assert mask.shape == (64, 1, 1) and mask.dtype == dtype
            assert torch.equal((x * mask).view(torch.uint8), out.view(torch.uint8))
            keep = 1 - p
            vals = set(mask.flatten().tolist())
            assert vals <= {0.0, float(torch.tensor(1.0, dtype=dtype).div_(keep))} if keep > 0 else vals == {0.0}
        # a rate that rounds the multiplier to exactly 1 in bf16 (block 2 of a depth-48 model)
        torch.manual_seed(0)
        m = DropPath(0.1 / 47).train().draw(torch.zeros(4096, 1, 1, dtype=torch.bfloat16))
        assert set(m.flatten().tolist()) <= {0.0, 1.0}
