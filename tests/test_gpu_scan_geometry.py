"""GPU: the launch geometry of the 32-channel-warp forward scan (scan_fwd_wp2_kernel) at the layer call of BASELINE config 2
(bs 64 x 1280 channels): a problem that fits one wave of 20 warps per SM runs as one CTA per SM holding the SM's whole share,
read back from the launch record of a torch.profiler trace (taken in a fresh process, the first profiler session of that process)."""
import json
import subprocess
import sys

import pytest

from util import ROOT

pytestmark = pytest.mark.gpu

WORKER = r"""
import json, os, sys, tempfile
sys.path.insert(0, sys.argv[1])
import torch
from torch.profiler import profile, ProfilerActivity
from zigma_b200 import selective_scan_fn, _lib
dev = "cuda"
Bt, E, L, N = 64, 1280, 64, 16
g = torch.Generator(device=dev).manual_seed(0)
u, z = torch.randn(Bt, L, E, device=dev, generator=g).bfloat16(), torch.randn(Bt, L, E, device=dev, generator=g).bfloat16()
dl = (0.5 * torch.rand(Bt, L, E, device=dev, generator=g)).bfloat16()
xbc = torch.randn(Bt, L, 2 * N, device=dev, generator=g).bfloat16()
A = -0.5 * torch.rand(E, N, device=dev, generator=g)
Dv, bias = torch.randn(E, device=dev, generator=g), torch.rand(E, device=dev, generator=g)
tr = lambda x: x.transpose(1, 2)
call = lambda: selective_scan_fn(tr(u), tr(dl), A, xbc[:, :, :N].permute(0, 2, 1).unsqueeze(1), xbc[:, :, N:].permute(0, 2, 1).unsqueeze(1),
                                 Dv, z=tr(z), delta_bias=bias, delta_softplus=True)
call()
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    call()
    torch.cuda.synchronize()
with tempfile.TemporaryDirectory() as d:
    path = os.path.join(d, "trace.json")
    prof.export_chrome_trace(path)
    ev = [e for e in json.load(open(path))["traceEvents"] if e.get("cat") == "kernel" and "scan_fwd" in e.get("name", "")]
print("RESULT " + json.dumps({"sms": torch.cuda.get_device_properties(0).multi_processor_count, "kernel": _lib.last_scan_kernel(),
                              "launches": [[e["name"], e["args"].get("grid"), e["args"].get("block")] for e in ev]}))
"""


def test_config2_scan_runs_one_cta_per_sm():
    p = subprocess.run([sys.executable, "-c", WORKER, ROOT], capture_output=True, text=True, timeout=600)
    line = [l for l in p.stdout.splitlines() if l.startswith("RESULT ")]
    assert p.returncode == 0 and line, p.stderr[-3000:]
    r = json.loads(line[0][7:])
    sms = r["sms"]
    if "scan_fwd_wp2_kernel" not in r["kernel"]:
        pytest.skip(f"this device ({sms} SMs) runs {r['kernel']} at config 2")
    assert len(r["launches"]) == 1 and "scan_fwd_wp2_kernel" in r["launches"][0][0], r
    _, grid, block = r["launches"][0]
    units = 64 * 1280 // 32
    warps = -(-units // sms)
    assert warps <= 20, (units, sms)
    assert block == [32 * warps, 1, 1] and grid == [-(-units // warps), 1, 1], r
    if sms == 132:
        assert block == [640, 1, 1] and grid == [128, 1, 1]
