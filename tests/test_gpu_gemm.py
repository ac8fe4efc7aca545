"""GPU (H100): the hand-written wgmma GEMM (zg_gemm_bf16_tn) against torch.matmul in fp32 on the same
bf16 operands, at the four projection shapes of the hot path and at ragged shapes."""
import pytest
import torch

from util import check_close

pytestmark = pytest.mark.gpu
DEV = "cuda"

SHAPES = [
    # M, N, K                      what
    (4096, 2560, 640),            # in_proj  (bs=4 slice of BASELINE config 2)
    (4096, 640, 1280),            # out_proj
    (4096, 72, 1280),             # x_proj   (N not a tile multiple)
    (4096, 1280, 40),             # dt_proj  (K < one k-block: TMA zero fill)
    (1000, 200, 136),             # everything ragged
    (128, 64, 64), (1, 8, 8), (129, 257, 72),
    (4096, 80, 1536), (4096, 768, 1536),   # x_proj / out_proj of the D = 768 models (80-wide tile; 3 x 256)
    (300, 5184, 72),              # 256-wide tiles whose last column tile holds 64 valid columns: its other chunks store nothing
    (300, 160, 64), (257, 150, 200), (520, 330, 96),   # 160-wide tiles: exact, ragged in N (tail columns by direct stores), two tiles + ragged
]


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("has_bias", [False, True])
def test_gemm_bf16_tn_matches_fp32_matmul(M, N, K, has_bias):
    from zigma_b200.gemm import linear_bf16
    torch.manual_seed(M + N + K)
    Kp = (K + 7) // 8 * 8
    a = torch.randn(M, Kp, device=DEV).bfloat16()[:, :K]       # leading dimension padded to a 16-byte pitch
    w = (torch.randn(N, Kp, device=DEV) / K ** 0.5).bfloat16()[:, :K]
    b = torch.randn(N, device=DEV).bfloat16() if has_bias else None
    out = linear_bf16(a, w, b)
    ref = a.float() @ w.float().t() + (b.float() if has_bias else 0)
    assert out.shape == (M, N) and out.dtype == torch.bfloat16
    check_close(out, ref, f"gemm {M}x{N}x{K} bias={has_bias}", rtol=8e-3, atol=1e-5, max_strict_viol=1.0)


def test_gemm_row_scatter_and_views():
    """out_rowmap scatters each batch's rows (out_proj + backward_permutation fused); A given as a
    column slice of a wider matrix (dt_proj reads x_dbl[:, :R] in place)."""
    from zigma_b200.gemm import linear_bf16
    import zigma_b200
    B, L, K, N = 3, 64, 72, 96
    x_dbl = torch.randn(B * L, K, device=DEV).bfloat16()
    w = torch.randn(N, 40, device=DEV).bfloat16()
    rev = torch.from_numpy(zigma_b200.reverse_permut_np(zigma_b200.zigzag_path(8)[2])).to(DEV)
    out = linear_bf16(x_dbl[:, :40], w, out_rowmap=rev.to(torch.int32), rows_per_batch=L)
    ref = (x_dbl[:, :40].float() @ w.float().t()).view(B, L, N)
    want = torch.empty_like(ref)
    want[:, rev] = ref                                   # row m lands at row rev[m]
    check_close(out.view(B, L, N), want, "gemm row scatter", rtol=8e-3, atol=1e-5, max_strict_viol=1.0)
    # the out_proj shape of the D = 640 models with the scatter (160-wide tiles, direct-store epilogue for every column)
    y = torch.randn(B * L, 128, device=DEV).bfloat16()
    w2 = (torch.randn(640, 128, device=DEV) / 128 ** 0.5).bfloat16()
    out2 = linear_bf16(y, w2, out_rowmap=rev.to(torch.int32), rows_per_batch=L)
    ref2 = (y.float() @ w2.float().t()).view(B, L, 640)
    want2 = torch.empty_like(ref2)
    want2[:, rev] = ref2
    check_close(out2.view(B, L, 640), want2, "gemm row scatter N=640", rtol=8e-3, atol=1e-5, max_strict_viol=1.0)


def test_engine_with_tcgen05_gemms(monkeypatch):
    """Whole bf16 model with the projections routed through zg_gemm_bf16_tn (ZIGMA_TCGEN05=1, the historical name of the switch) == library-GEMM engine."""
    from oracle import synth
    from oracle.gen_golden import model_io
    from util import model_case
    from zigma_b200 import ZigMa
    g, cfg, shapes = model_case("tiny_zigzag8_bf16")
    outs = {}
    for flag in ("0", "1"):
        monkeypatch.setenv("ZIGMA_TCGEN05", flag)
        m = ZigMa(device=DEV, dtype=torch.bfloat16, **cfg).eval()
        m.load_state_dict(synth.synth_state_dict(shapes, seed=0, dtype=torch.bfloat16))
        x, tt, _ = model_io(cfg, 2)
        with torch.no_grad():
            outs[flag] = m(x.to(DEV).bfloat16(), tt.to(DEV).bfloat16()).float()
    check_close(outs["1"], outs["0"], "engine wgmma vs library GEMMs", rtol=3e-2, atol=3e-2, scale_atol=False, max_strict_viol=1.0)
    check_close(outs["1"], g["out"], "engine wgmma vs reference bf16", rtol=5e-2, atol=5e-2, scale_atol=False, max_strict_viol=1.0)
