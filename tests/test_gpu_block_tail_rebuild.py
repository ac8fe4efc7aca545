"""GPU: the block tail that rebuilds its x from the previous tail's residual_out, rstd and norm_w (zg_block_tail_fwd_rebuild) equals,
bit for bit, the plain tail fed the previous tail's normed output -- every instantiation (dtypes, both row buckets), with and
without a row table, with the spatial-video fold (mod_div) and as the final layer; residual_out, modded, rstd and normed alike."""
import itertools

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dtype,D,rowmap,fold,final", [
    (dt, D, rm, fold, final) for dt, D, rm, fold, final in itertools.product(
        (torch.float32, torch.float16, torch.bfloat16), (256, 640, 1024), (False, True), (1, 4), (False, True))])
def test_rebuild_equals_plain_tail_on_previous_normed(dtype, D, rowmap, fold, final):
    from zigma_b200.engine import block_tail
    dev = "cuda"
    B, L, eps = 3, 64, 1e-5
    g = torch.Generator(device=dev).manual_seed(D + 7 * fold + 3 * rowmap + int(final))
    rnd = lambda *s: torch.randn(*s, device=dev, generator=g)
    # the previous tail (plain entry): its residual_out, normed and rstd
    mods0, mods1 = rnd(B, 3 * D).to(dtype), rnd(B, 3 * D).to(dtype)
    w0, w1 = (1 + 0.3 * rnd(D)).to(dtype), (1 + 0.3 * rnd(D)).to(dtype)
    r0, n0, _, rs0 = block_tail(rnd(B, L, D).to(dtype), rnd(B, L, D).to(dtype), mods0[:, :D], mods0[:, D:2 * D], mods0[:, 2 * D:], w0,
                                4 * rnd(B, L, D), None, eps, want_rstd=True)
    # this tail: (B fold, L / fold) rows of the same memory with fold != 1, as the spatial video layers call it
    Bf, Lf = B * fold, L // fold
    mix = rnd(Bf, Lf, D).to(dtype)
    perm = torch.randperm(Lf, device=dev, generator=g).to(torch.int32) if rowmap else None
    shift, scale = (None, None) if final else (mods1[:, D:2 * D], mods1[:, 2 * D:])
    args = (mix, mods1[:, :D], shift, scale, w1, r0.view(Bf, Lf, D), perm, eps)
    want = block_tail(n0.view(Bf, Lf, D), *args, final=final, mod_div=fold, want_rstd=True)
    got = block_tail(None, *args, final=final, mod_div=fold, want_rstd=True, x_from=(rs0, w0))
    names = ("residual_out", "normed", "modded", "rstd")
    for name, a, b in zip(names, got, want):
        if name == "normed" and not final:
            assert a is None
            continue
        assert (a is None) == (b is None), name
        if a is not None:
            bits = lambda t: t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)
            assert torch.equal(bits(a), bits(b)), name
