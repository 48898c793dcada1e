"""GPU: the persistent warp-specialised 128x256 GEMM (ttb_gemm variant 7, the default for problems of at least one wave
of 128x128 tiles) against the one-tile kernel (variant 1) and the SIMT checker (force_ref).

Both wgmma kernels add the same k16 products in the same order and finish every 32x32 block with the same epilogue
code, so variant 7 must reproduce variant 1 bit for bit: outputs and GroupNorm partials. The SIMT checker sums in
another order; it is held to fp32 accumulation noise relative to the output scale."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _mk(shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).cuda()


def _run(variant, *, M, N, K, taps=1, batch=1, act=0, bias=True, residual=None, inplace=False, out="f32", ldob=None,
         bcast=False, gn=False, tap_dilation=1, w_static=False, force_ref=False, seed=0):
    """One ttb_gemm call on seeded operands; returns (out_f32, out_bf16, gn partials), each possibly None."""
    from tortoise_tts_b200 import lib
    rows = M
    A = _mk((1 if bcast else batch, rows, K), 1.0, seed).to(torch.bfloat16)
    W = _mk((N, taps * K), (taps * K) ** -0.5, seed + 1).to(torch.bfloat16)
    b = _mk((N,), 0.5, seed + 2) if bias else None
    n_out = N // 2 if act == lib.ACT_GEGLU else N
    res = _mk((batch, M, n_out), 1.0, seed + 3) if residual else None
    of = None
    if out in ("f32", "both"):
        of = res.clone() if inplace else torch.full((batch, M, n_out), float("nan"), device="cuda")
    ob = None
    ldob = n_out if ldob is None else ldob
    if out in ("bf16", "both"):
        ob = torch.zeros((batch, M, ldob), device="cuda", dtype=torch.bfloat16)
    part = lib.groupnorm_scratch(batch, N // 32, "cuda") if gn else None
    pad = tap_dilation * (taps - 1) // 2
    lib.gemm(A, W, M=M, N=N, K=K, taps=taps, pad=pad, batch=batch, bias=b,
             residual=(of if inplace else res), out_f32=of, out_bf16=ob, rows=rows, a_bstride=0 if bcast else rows * K,
             res_bstride=M * n_out, outf_bstride=M * n_out, outb_bstride=M * ldob, ldob=ldob, act=act,
             variant=variant, force_ref=force_ref, gn_partials=part, gn_groups=N // 32 if gn else 0,
             tap_dilation=tap_dilation, w_static=w_static)
    torch.cuda.synchronize()
    return of, ob, part


def _lib():
    from tortoise_tts_b200 import lib
    return lib


# name -> kwargs of _run
CASES = {
    "diff_conv1x1": dict(M=1872, N=1024, K=1024, batch=2, residual=True, inplace=True, gn=True),
    "diff_conv_k3": dict(M=1872, N=1024, K=1024, taps=3, batch=2, residual=True, inplace=True, gn=True),
    "diff_qkv_bf16": dict(M=1872, N=3072, K=1024, batch=2, out="bf16", bias=False),
    "cat_ldob_2c": dict(M=1872, N=1024, K=1024, batch=2, out="bf16", ldob=2048),
    "bcast_a_bstride0": dict(M=1872, N=1024, K=1024, batch=2, bcast=True, out="both"),
    "integrating_k2048": dict(M=1872, N=1024, K=2048, batch=2),
    "out_conv_n200": dict(M=1872, N=200, K=1024, taps=3, batch=2),
    "clvp_qkv": dict(M=27520, N=2304, K=768, out="bf16"),
    "clvp_geglu": dict(M=27520, N=6144, K=768, act="GEGLU", out="bf16"),
    "vocoder_kpred": dict(M=1720, N=2304, K=64, taps=3, act="LRELU02"),
    "tap_dilation": dict(M=2000, N=512, K=512, taps=3, tap_dilation=3, residual=True),
    "m_below_tile": dict(M=100, N=512, K=256, out="both"),
    "ragged_tile_count": dict(M=1000, N=768, K=320, batch=3, act="SILU"),    # 8 x 3 x 3 = 72 tiles
    "tiles_over_grid": dict(M=5000, N=1280, K=256, act="GELU_ERF"),          # 40 x 5 = 200 tiles on 132 SMs
    "w_static": dict(M=1872, N=1024, K=1024, taps=3, batch=2, w_static=True, residual=True),
}


def _case(name):
    kw = dict(CASES[name])
    if "act" in kw:
        kw["act"] = getattr(_lib(), "ACT_" + kw["act"])
    return kw


@pytest.mark.parametrize("name", list(CASES))
def test_ws_bit_identical_to_one_tile(name):
    kw = _case(name)
    got = _run(7, **kw)
    want = _run(1, **kw)
    for g, w, what in zip(got, want, ("out_f32", "out_bf16", "gn_partials")):
        assert (g is None) == (w is None)
        if g is not None:
            assert not torch.isnan(g).any(), what
            assert torch.equal(g, w), "%s: max |diff| %.3e" % (what, (g.float() - w.float()).abs().max().item())


@pytest.mark.parametrize("name", [n for n in CASES if not CASES[n].get("gn") and CASES[n].get("tap_dilation", 1) == 1
                                  and n != "clvp_geglu"])
def test_ws_against_simt_checker(name):
    kw = _case(name)
    got = _run(7, **kw)
    want = _run(0, force_ref=True, **kw)
    for g, w, what in zip(got, want, ("out_f32", "out_bf16")):
        if g is None:
            continue
        g, w = g.float(), w.float()
        scale = w.abs().max().item()
        tol = (8e-3 if what == "out_bf16" else 2e-3) * scale
        err = (g - w).abs().max().item()
        assert err <= tol, "%s: max |diff| %.3e > %.3e" % (what, err, tol)


def test_ws_is_default_for_one_wave():
    """Variant 0 at the diffusion k=3 shape takes the warp-specialised kernel: bit-identical to forcing variant 7."""
    kw = _case("diff_conv_k3")
    got = _run(0, **kw)
    want = _run(7, **kw)
    for g, w in zip(got, want):
        assert (g is None and w is None) or torch.equal(g, w)


def test_ws_rejects_splitk():
    lib = _lib()
    A = torch.zeros(1, 256, 256, device="cuda", dtype=torch.bfloat16)
    W = torch.zeros(256, 256, device="cuda", dtype=torch.bfloat16)
    out = torch.zeros(2, 256, 256, device="cuda")
    with pytest.raises(lib.TtbError):
        lib.gemm(A, W, M=256, N=256, K=256, out_f32=out, outf_bstride=256 * 256, splitk=2, variant=7)
