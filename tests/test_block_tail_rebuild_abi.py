"""CPU: the block tail that rebuilds its x (zg_block_tail_fwd_rebuild) -- ctypes layout, export, the argument checks on empty
batches (nothing can launch), and a SASS audit of the built library: every block-tail kernel that existed before it compiles to the
same instructions, the new instantiations and the forward-scan kernels of 32-channel warps stay inside their register budgets."""
import ctypes as C
import hashlib
import json
import os
import re
import subprocess
import tempfile

import pytest

from util import ROOT, GOLD

HEADER = os.path.join(ROOT, "include", "zigma_b200.h")
OBJ = os.path.join(ROOT, "build", "obj")
FAKE = 1 << 20            # stands in for device pointers: the checks read addresses (alignment) only, never memory


def _built():
    import __graft_entry__
    __graft_entry__.build()
    from zigma_b200 import _lib
    return _lib


def _tool(name):
    for d in (os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin"), "/usr/local/cuda/bin"):
        if os.path.exists(os.path.join(d, name)):
            return os.path.join(d, name)
    pytest.skip(f"{name} not found")


def test_ctypes_layout_matches_c():
    from zigma_b200 import _lib
    st, cname = _lib.BlockTailRebuildParams, "zg_block_tail_rebuild_params"
    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{HEADER}"', "int main(void) {",
             f'printf("{cname} %zu\\n", sizeof({cname}));']
    lines += [f'printf("{cname}.{f} %zu\\n", offsetof({cname}, {f}));' for f, _ in st._fields_]
    lines.append("return 0; }")
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "l.c"), os.path.join(d, "l")
        open(src, "w").write("\n".join(lines))
        subprocess.check_call(["gcc", "-o", exe, src])
        out = subprocess.check_output([exe]).decode().split("\n")
    c_layout = dict(l.split() for l in out if l)
    assert int(c_layout[cname]) == C.sizeof(st)
    for f, _ in st._fields_:
        assert int(c_layout[f"{cname}.{f}"]) == getattr(st, f).offset, f
    assert st.x_rstd.offset == C.sizeof(_lib.BlockTailParams)


def test_declared_and_exported():
    _lib = _built()
    declared = set(re.findall(r"\b(zg_[a-z0-9_]+)\s*\(", open(HEADER).read()))
    l = _lib.lib()
    assert "zg_block_tail_fwd_rebuild" in declared and "zg_block_tail_fwd_rebuild" in _lib.EXPORTS
    assert hasattr(l, "zg_block_tail_fwd_rebuild") and _lib.EXPORTS.index("zg_block_tail_fwd_rebuild") >= 5
    assert l.zg_abi_version() == 5


def _params(_lib, dtype=None, dim=640, final=False):
    """Valid params of an EMPTY batch (batch 0): every check runs before the empty-batch return."""
    dtype = _lib.ZG_BF16 if dtype is None else dtype
    q = _lib.BlockTailRebuildParams()
    p = q.base
    for i, n in enumerate(["mix", "norm_w", "residual", "residual_out", "modded", "rowmap"]):
        setattr(p, n, FAKE * (i + 1))
    p.normed = FAKE * 16 if final else None
    esz = 4 if dtype == _lib.ZG_F32 else 2
    p.shift, p.scale, p.gate = FAKE * 64, FAKE * 64 + dim * esz, FAKE * 64 + 2 * dim * esz
    p.mod_rs = 3 * dim
    p.batch, p.seqlen, p.dim, p.dtype, p.eps, p.final_layer = 0, 16, dim, dtype, 1e-5, int(final)
    q.x_rstd, q.x_norm_w = FAKE * 128, FAKE * 130
    return q


def _call(_lib, q):
    l = _lib.lib()
    rc = l.zg_block_tail_fwd_rebuild(C.byref(q), C.c_void_p(None))
    return rc, l.zg_last_error().decode()


def test_accepts_and_rejects_on_empty_batches():
    _lib = _built()
    for dt in (_lib.ZG_F32, _lib.ZG_F16, _lib.ZG_BF16):
        for dim in (36, 368, 640, 1024):
            for final in (False, True):
                rc, err = _call(_lib, _params(_lib, dt, dim, final))
                assert rc == 0, (dt, dim, final, err)

    def rejected(what, **kw):
        q = _params(_lib)
        for k, v in kw.items():
            setattr(q if k in ("x_rstd", "x_norm_w") else q.base, k, v)
        rc, err = _call(_lib, q)
        assert rc != 0, what
        return err

    assert "x must be NULL" in rejected("x given", x=FAKE * 32)
    assert "residual" in rejected("no residual", residual=None)
    assert "x_rstd" in rejected("no x_rstd", x_rstd=None)
    assert "x_norm_w" in rejected("no x_norm_w", x_norm_w=None)
    assert "final_layer needs normed" in rejected("final without normed", final_layer=1)
    assert "1024" in rejected("dim above 1024", dim=1536)
    assert "aligned" in rejected("x_norm_w 2 bytes off", x_norm_w=FAKE * 130 + 2)
    assert "aligned" in rejected("x_rstd 2 bytes off", x_rstd=FAKE * 128 + 2)
    # what the plain entry point rejects
    assert "multiple of 4" in rejected("dim 38", dim=38)
    assert "16-byte" in rejected("residual misaligned", residual=FAKE * 3 + 8)
    assert "mix needs gate" in rejected("mix without gate", gate=None)
    assert "null" in rejected("no norm_w", norm_w=None)


def _sass(obj):
    """{function: sha1 of its SASS without the instruction addresses} of a cubin object."""
    out = subprocess.run([_tool("cuobjdump"), "-sass", obj], capture_output=True, text=True, check=True).stdout
    fs, cur = {}, None
    for l in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", l)
        if m:
            cur = m.group(1)
            fs[cur] = []
        elif cur:
            fs[cur].append(re.sub(r"/\*[0-9a-f]{4}\*/", "", l).strip())
    return {k: hashlib.sha1("\n".join(v).encode()).hexdigest() for k, v in fs.items()}


def _res_usage(obj):
    out = subprocess.run([_tool("cuobjdump"), "-res-usage", obj], capture_output=True, text=True, check=True).stdout
    return {m.group(1): (int(m.group(2)), int(m.group(3)), int(m.group(4)))
            for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)}


def test_existing_block_tail_kernels_keep_their_sass():
    """The rebuild variant is a new instantiation of the shared four-warps-per-row body: every block-tail kernel compiled before it
    (forward and backward, all dtypes and row buckets; hashes recorded with CUDA 12.9) is instruction for instruction unchanged."""
    _built()
    want = json.load(open(os.path.join(GOLD, "block_tail_sass_sha1.json")))
    got = _sass(os.path.join(OBJ, "norm.o"))
    changed = [f for f in want if got.get(f) != want[f]]
    assert not changed, changed


def test_register_budgets():
    """scan_fwd_wp2_kernel: 96 registers, no stack or local memory -- the cap of its 640-thread launch bound, and what lets 21 warps stay
    resident per SM.  The rebuild tail: within the 40 registers of ZG_TAIL_MINB = 12 CTAs per SM, and no local memory in the 16-bit
    instantiations (fp32 at dim > 512 spills less than the plain fp32 kernel it replaces)."""
    _built()
    for tu in ("scan_fwd_wp2_bf16.o", "scan_fwd_wp2_f16.o"):
        use = {k: v for k, v in _res_usage(os.path.join(OBJ, tu)).items() if "scan_fwd_wp2_kernel" in k}
        assert len(use) == 2, use
        for k, (reg, stack, local) in use.items():
            assert (reg, stack, local) == (96, 0, 0), (k, reg, stack, local)
    norm = _res_usage(os.path.join(OBJ, "norm.o"))
    rb = {k: v for k, v in norm.items() if "block_tail_rebuild_fwd_kernel" in k}
    assert len(rb) == 6, rb
    for k, (reg, stack, local) in rb.items():
        assert reg <= 40, (k, reg)
        if "kernelIf" not in k:
            assert stack == 0 and local == 0, (k, stack, local)
        else:
            plain = norm[k.replace("29block_tail_rebuild_fwd_kernel", "22block_tail_row4_kernel").replace("EEEv28zg_block_tail_rebuild_params", "ELb0EEEv20zg_block_tail_params")]
            assert local == 0 and stack <= plain[1], (k, stack, local, plain)
