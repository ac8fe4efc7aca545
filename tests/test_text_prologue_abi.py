"""CPU: the text-prologue entry points (zg_text_prologue_fwd, zg_text_prologue_bwd and its _det twin) -- ctypes layout,
exports, the argument checks on empty batches (nothing can launch), the deterministic workspace size, and a SASS audit of
the built library (the exact instantiation sets, no floating-point atomic in the DET ones, every other kernel of norm.cu
compiled to the code it had before the prologue existed)."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import pytest

from util import ROOT

HEADER = os.path.join(ROOT, "include", "zigma_b200.h")
FAKE = 1 << 20            # stands in for device pointers: the checks read addresses (alignment) only, never memory
NEW_FUNCS = ("zg_text_prologue_fwd", "zg_text_prologue_bwd", "zg_text_prologue_bwd_det", "zg_text_prologue_bwd_det_workspace_bytes")


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
    structs = {"zg_text_prologue_params": _lib.TextPrologueParams, "zg_text_prologue_bwd_params": _lib.TextPrologueBwdParams}
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


def test_declared_and_exported():
    _lib = _built()
    declared = set(re.findall(r"\b(zg_[a-z0-9_]+)\s*\(", open(HEADER).read()))
    l = _lib.lib()
    for n in NEW_FUNCS:
        assert n in declared and n in _lib.EXPORTS and hasattr(l, n), n
    assert "zg_text_prologue_bwd" in _lib.DET_OPS
    assert l.zg_abi_version() == 5


def _fwd(_lib, dtype=None, dim=768):
    """Valid forward params of an EMPTY batch (batch 0): every check runs before the empty-batch return."""
    dtype = _lib.ZG_BF16 if dtype is None else dtype
    p = _lib.TextPrologueParams()
    _ptrs(p, ["x", "mix", "rowmap", "hidden", "q_in", "mean", "rstd"])
    esz = 4 if dtype == _lib.ZG_F32 else 2
    p.gate, p.shift, p.scale = FAKE * 64, FAKE * 64 + dim * esz, FAKE * 64 + 2 * dim * esz
    p.mod_rs = 6 * dim
    p.batch, p.seqlen, p.dim, p.dtype, p.eps = 0, 16, dim, dtype, 1e-6
    return p


def _bwd(_lib, dtype=None, dim=768, nparts=1):
    dtype = _lib.ZG_BF16 if dtype is None else dtype
    p = _lib.TextPrologueBwdParams()
    _ptrs(p, ["d_hidden", "d_q", "hidden", "mix", "mean", "rstd", "rowmap", "d_x", "d_mix", "dgate", "dshift", "dscale"])
    esz = 4 if dtype == _lib.ZG_F32 else 2
    p.gate, p.scale = FAKE * 64, FAKE * 64 + 2 * dim * esz
    p.mod_rs = 6 * dim
    p.batch, p.seqlen, p.dim, p.dtype, p.nparts = 0, 16, dim, dtype, nparts
    return p


def _call(_lib, name, q, ws=None, ws_bytes=0):
    l = _lib.lib()
    if name.endswith("_det"):
        rc = getattr(l, name)(C.byref(q), C.c_void_p(ws), C.c_int64(ws_bytes), C.c_void_p(None))
    else:
        rc = getattr(l, name)(C.byref(q), C.c_void_p(None))
    return rc, l.zg_last_error().decode()


def test_forward_accepts_and_rejects_on_empty_batches():
    _lib = _built()
    for dt in (_lib.ZG_F32, _lib.ZG_F16, _lib.ZG_BF16):
        for dim in (4, 64, 368, 768, 1024, 1536, 2048):
            rc, err = _call(_lib, "zg_text_prologue_fwd", _fwd(_lib, dt, dim))
            assert rc == 0, (dt, dim, err)
    q = _fwd(_lib)
    q.rowmap = q.mean = q.rstd = None
    assert _call(_lib, "zg_text_prologue_fwd", q)[0] == 0, "rowmap / mean / rstd are optional"

    def rejected(what, dtype=None, **kw):
        q = _fwd(_lib, dtype)
        for k, v in kw.items():
            setattr(q, k, v)
        rc, err = _call(_lib, "zg_text_prologue_fwd", q)
        assert rc != 0, what
        return err

    for n in ("x", "mix", "gate", "shift", "scale", "hidden", "q_in"):
        assert "null" in rejected(f"null {n}", **{n: None})
    assert "multiple of 4" in rejected("dim 38", dim=38)
    assert "2048" in rejected("dim above 2048", dim=2052)
    assert "multiple of 4" in rejected("dim 0", dim=0)
    assert "stride" in rejected("mod_rs 6", mod_rs=6)
    assert "16-byte" in rejected("x misaligned", x=FAKE + 8)
    assert "16-byte" in rejected("mix misaligned", mix=FAKE * 2 + 4)
    assert "16-byte" in rejected("q_in misaligned", q_in=FAKE * 5 + 8)
    assert "aligned" in rejected("gate 2 bytes off", gate=FAKE * 64 + 2)
    assert "aligned" in rejected("fp32 scale 8 bytes off", dtype=_lib.ZG_F32, scale=FAKE * 64 + 8)
    assert "dtype" in rejected("bad dtype", dtype=7)
    assert "negative" in rejected("negative batch", batch=-1)


@pytest.mark.parametrize("name", ["zg_text_prologue_bwd", "zg_text_prologue_bwd_det"])
def test_backward_accepts_and_rejects_on_empty_batches(name):
    _lib = _built()
    for dt in (_lib.ZG_F32, _lib.ZG_F16, _lib.ZG_BF16):
        for dim in (4, 64, 368, 640, 768, 1024):
            rc, err = _call(_lib, name, _bwd(_lib, dt, dim))
            assert rc == 0, (name, dt, dim, err)
    q = _bwd(_lib)
    q.d_hidden = q.rowmap = q.dgate = q.dshift = q.dscale = None
    assert _call(_lib, name, q)[0] == 0, "d_hidden / rowmap / column sums are optional"

    def rejected(what, **kw):
        q = _bwd(_lib)
        for k, v in kw.items():
            setattr(q, k, v)
        rc, err = _call(_lib, name, q)
        assert rc != 0, what
        return err

    for n in ("d_q", "hidden", "mix", "gate", "scale", "mean", "rstd", "d_x", "d_mix"):
        assert "null" in rejected(f"null {n}", **{n: None})
    assert "1024" in rejected("dim above 1024", dim=1028)
    assert "1024" in rejected("dim 1536 (forward only)", dim=1536)
    assert "multiple of 4" in rejected("dim 38", dim=38)
    assert "nparts" in rejected("nparts 0", nparts=0)
    assert "nparts" in rejected("nparts 65536", nparts=65536)
    assert "16-byte" in rejected("d_hidden misaligned", d_hidden=FAKE + 2)
    assert "16-byte" in rejected("d_mix misaligned", d_mix=FAKE * 9 + 8)
    assert "aligned" in rejected("gate 2 bytes off", gate=FAKE * 64 + 2)


def test_det_needs_a_warp_per_batch_element_and_a_workspace():
    """With rows to do, the _det twin rejects nparts with 4 * nparts < batch and a workspace below the query, and launches
    nothing (the pointers are fake: a launch would fault)."""
    _lib = _built()
    q = _bwd(_lib, nparts=1)
    q.batch = 5
    rc, err = _call(_lib, "zg_text_prologue_bwd_det", q)
    assert rc != 0 and "4 * nparts >= batch" in err
    q.nparts = 2
    need = _lib.det_workspace_bytes("zg_text_prologue_bwd", q)
    assert need > 0
    rc, err = _call(_lib, "zg_text_prologue_bwd_det", q, ws=FAKE * 256, ws_bytes=need - 16)
    assert rc != 0 and "workspace" in err
    rc, err = _call(_lib, "zg_text_prologue_bwd_det", q, ws=FAKE * 256 + 8, ws_bytes=need)
    assert rc != 0 and "workspace" in err, "misaligned workspace"


def test_det_workspace_bytes_formula():
    """(4 nparts / batch) partial rows of batch * dim fp32 per non-NULL column sum, each region rounded up to 16 bytes; the
    block tail's query on the same shape gives the same number."""
    _lib = _built()
    for B in (1, 3, 16, 64):
        for L in (1, 37, 1024):
            for D in (4, 36, 768, 1024):
                for nparts in (max(1, (B + 3) // 4), 7, 256):
                    for absent in ((), ("dshift",), ("dgate", "dscale")):
                        q = _bwd(_lib, dim=D, nparts=nparts)
                        q.batch, q.seqlen = B, L
                        for n in absent:
                            setattr(q, n, None)
                        region = ((4 * nparts // B) * B * D * 4 + 15) // 16 * 16
                        assert _lib.det_workspace_bytes("zg_text_prologue_bwd", q) == (3 - len(absent)) * region, (B, L, D, nparts, absent)
                        t = _lib.BlockTailBwdParams()
                        _ptrs(t, ["r", "rstd", "norm_w", "d_x", "d_norm_w", "mix", "gate", "d_mix", "scale"])
                        t.dgate, t.dshift, t.dscale = q.dgate, q.dshift, q.dscale
                        t.batch, t.seqlen, t.dim, t.nparts = B, L, D, nparts
                        assert _lib.det_workspace_bytes("zg_block_tail_bwd", t) == _lib.det_workspace_bytes("zg_text_prologue_bwd", q)
    q = _bwd(_lib)
    assert _lib.det_workspace_bytes("zg_text_prologue_bwd", q) == 0, "empty batch"


def _sass_functions(path):
    from test_deterministic_abi import _tool
    cuobjdump, filt = _tool("cuobjdump"), _tool("cu++filt")
    if cuobjdump is None or filt is None:
        pytest.skip("cuobjdump / cu++filt not available")
    sass = subprocess.run([cuobjdump, "-sass", path], check=True, capture_output=True, text=True).stdout
    funcs, cur = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur is not None and re.search(r"/\*[0-9a-f]{4}\*/", line):
            funcs[cur].append(re.sub(r"\s+", " ", line.strip()))
    names = list(funcs)
    demangled = subprocess.run([filt], input="\n".join(names), check=True, capture_output=True, text=True).stdout.splitlines()
    return funcs, dict(zip(names, demangled))


def test_sass_text_prologue_instantiations():
    """12 forward (T x Q 1/2/3/4) and 24 backward (T x MAXQ 4/5/6/8 x DET) instantiations; no floating-point atomic or
    reduction in the 12 DET ones."""
    from test_deterministic_abi import FLOAT_ATOMIC
    _lib = _built()
    funcs, dem = _sass_functions(_lib.LIB_PATH)
    fwd, bwd, det = set(), set(), 0
    for mangled, d in dem.items():
        m = re.search(r"zg::(text_prologue_(?:fwd|bwd)_kernel)<(.*)>\(", d)
        if m is None:
            continue
        args = tuple({"(bool)1": "true", "(bool)0": "false"}.get(a.strip(), a.strip()) for a in m.group(2).split(","))
        args = tuple(re.sub(r"^\((?:int|unsigned int)\)", "", a) for a in args)
        if m.group(1) == "text_prologue_fwd_kernel":
            fwd.add(args)
        else:
            bwd.add(args)
            if args[-1] == "true":
                det += 1
                bad = [l for l in funcs[mangled] if FLOAT_ATOMIC.search(l)]
                assert not bad, f"{d}: {bad[:3]}"
    T = ("float", "__half", "__nv_bfloat16")
    assert fwd == {(t, q) for t in T for q in ("1", "2", "3", "4")}
    assert bwd == {(t, q, d) for t in T for q in ("4", "5", "6", "8") for d in ("false", "true")}
    assert det == 12


def test_sass_of_the_other_norm_kernels_unchanged():
    """norm.cu compiled without the text prologue (the same file with its kernels, launchers and entry points cut out) and
    as built: every kernel the two objects share has the same instructions, and the built one adds only text_prologue_*."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    csrc = os.path.join(ROOT, "zigma_b200", "csrc")
    src = open(os.path.join(csrc, "norm.cu")).read()
    begin = src.index("// Text prologue (see include/zigma_b200.h)")
    begin = src.rindex("// ----", 0, begin)
    end = src.index("template <typename T, typename R> static int norm_fwd_tr")
    tail = src.index("static int text_prologue_fwd_validate")
    without = src[:begin] + src[end:tail]
    assert "text_prologue" not in without
    with tempfile.TemporaryDirectory() as d:
        objs, procs = {}, []
        for tag, text in (("with", src), ("without", without)):
            cu = os.path.join(d, tag + ".cu")
            open(cu, "w").write(text)
            objs[tag] = os.path.join(d, tag + ".o")
            procs.append(subprocess.Popen([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler",
                                           "-fPIC", "-I", csrc, "-c", cu, "-o", objs[tag]], stdout=subprocess.DEVNULL, stderr=subprocess.PIPE))
        for pr in procs:
            assert pr.wait() == 0, pr.stderr.read().decode()[-2000:]
        a, _ = _sass_functions(objs["without"])
        b, dem = _sass_functions(objs["with"])
    assert len(a) > 100
    changed = [n for n in a if a[n] != b.get(n)]
    assert not changed, changed[:5]
    added = [dem[n] for n in b if n not in a]
    assert added and all("text_prologue" in n for n in added), added[:5]
