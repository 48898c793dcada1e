"""GPU: the wgmma GEMM / conv-as-GEMM (ttb_gemm) against a plain PyTorch fp32 reference of the same op on the
same bf16-rounded operands (tolerance: fp32 accumulation-order noise, 2e-3 relative to the output scale), and the
SIMT checker kernel against the same reference."""
import pytest
import torch
import torch.nn.functional as F

from gpu_util import report

pytestmark = pytest.mark.gpu


def _mk(shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).cuda()


def _run(M, N, K, taps=1, batch=1, act=0, bias=True, residual=False, out="f32", tile_n=0, force_ref=False, seed=0,
         variant=0):
    from tortoise_tts_b200 import lib
    A = _mk((batch, M, K), 1.0, seed).to(torch.bfloat16)
    W = _mk((N, taps, K), K ** -0.5, seed + 1).to(torch.bfloat16)
    b = _mk((N,), 0.5, seed + 2) if bias else None
    n_out = N // 2 if act == lib.ACT_GEGLU else N
    res = _mk((batch, M, n_out), 1.0, seed + 3) if residual else None
    of = torch.full((batch, M, n_out), float("nan"), device="cuda") if out in ("f32", "both") else None
    ob = torch.zeros((batch, M, n_out), device="cuda", dtype=torch.bfloat16) if out in ("bf16", "both") else None
    lib.gemm(A, W.reshape(N, taps * K), M=M, N=N, K=K, taps=taps, pad=(taps - 1) // 2, batch=batch, bias=b,
             residual=res, out_f32=of, out_bf16=ob, a_bstride=M * K, res_bstride=M * n_out, outf_bstride=M * n_out,
             outb_bstride=M * n_out, act=act, tile_n=tile_n, force_ref=force_ref, variant=variant)
    torch.cuda.synchronize()
    # reference: plain fp32 matmuls on the CPU (no cuDNN / TF32 involved): conv over tokens == sum of shifted GEMMs
    a, w = A.float().cpu(), W.float().cpu()
    y = torch.zeros(batch, M, N)
    pad = (taps - 1) // 2
    for tap in range(taps):
        sh = tap - pad
        lo, hi = max(0, -sh), min(M, M - sh)
        y[:, lo:hi] += a[:, lo + sh:hi + sh] @ w[:, tap].t()
    if b is not None:
        y = y + b.cpu()
    y = y.cuda()
    if act == lib.ACT_GELU_NEW:
        y = F.gelu(y, approximate="tanh")
    elif act == lib.ACT_SILU:
        y = F.silu(y)
    elif act == lib.ACT_LRELU02:
        y = F.leaky_relu(y, 0.2)
    elif act == lib.ACT_GEGLU:
        y = y[..., 0::2] * F.gelu(y[..., 1::2])
    if residual:
        y = y + res
    return y, of, ob


CASES = [
    dict(M=128, N=128, K=64),
    dict(M=128, N=128, K=64, tile_n=64),
    dict(M=128, N=256, K=256, tile_n=128),
    dict(M=300, N=200, K=128),                       # M and N tails
    dict(M=1, N=8194, K=128),                        # lm-head at M=1
    dict(M=256, N=3072, K=1024, out="bf16"),         # AR c_attn at B=256
    dict(M=256, N=1024, K=4096, residual=True),      # AR mlp.c_proj (+residual)
    dict(M=256, N=4096, K=1024, act=1, out="bf16"),  # c_fc + gelu_new
    dict(M=333, N=256, K=128, taps=3, batch=2, residual=True),  # conv k=3, batch boundaries
    dict(M=374, N=1024, K=1024, taps=3, batch=2, tile_n=128),
    dict(M=150, N=512, K=128, act=3, out="bf16"),    # GEGLU
    dict(M=77, N=200, K=1024, taps=3),               # diffusion out conv (N=200)
    dict(M=1882, N=24832, K=64, taps=3),             # UnivNet kernel predictor
    dict(M=130, N=192, K=64, act=2, out="both"),
    dict(M=1872, N=1024, K=1024, taps=3, batch=2, tile_n=256, residual=True),   # 128x256 tiles
    dict(M=3000, N=2304, K=768, out="bf16"),                                     # auto -> 128x256 (CLVP qkv shape)
    dict(M=300, N=512, K=128, tile_n=256, act=1),
]


@pytest.mark.parametrize("case", CASES, ids=[str(i) for i in range(len(CASES))])
def test_gemm_tcgen05(case):
    y, of, ob = _run(**case)
    scale = y.abs().max().item()
    if of is not None:
        err = (of - y).abs().max().item()
        report("gemm_tc_f32 %s" % case, err / scale)
        assert err / scale < 2e-3, (err, scale)
    if ob is not None:
        err = (ob.float() - y).abs().max().item()
        report("gemm_tc_bf16 %s" % case, err / scale)
        assert err / scale < 1e-2, (err, scale)


@pytest.mark.parametrize("M,N,K,tile_n,splitk", [(256, 1024, 1024, 32, 2), (256, 1024, 4096, 32, 4), (256, 3072, 1024, 32, 1),
                                                 (100, 128, 128, 32, 2), (256, 1024, 4096, 64, 3)])
def test_gemm_skinny_splitk(M, N, K, tile_n, splitk):
    """Decode-shape GEMMs: 32-column tiles and split-K partials whose fixed-order sum equals the full product."""
    from tortoise_tts_b200 import lib
    A = _mk((M, K), 1.0, 5).to(torch.bfloat16)
    W = _mk((N, K), K ** -0.5, 6).to(torch.bfloat16)
    want = (A.float().cpu() @ W.float().cpu().t()).cuda()
    if splitk == 1:
        b = _mk((N,), 0.5, 7)
        out = torch.empty(M, N, device="cuda")
        lib.gemm(A, W, M=M, N=N, K=K, bias=b, out_f32=out, tile_n=tile_n)
        got = out - b
    else:
        kb = K // 64
        per = (kb + splitk - 1) // splitk
        nz = (kb + per - 1) // per
        part = torch.full((nz, M, N), float("nan"), device="cuda")
        lib.gemm(A, W, M=M, N=N, K=K, out_f32=part, outf_bstride=M * N, tile_n=tile_n, splitk=splitk)
        got = part.sum(dim=0)
        # and through the fused residual + LayerNorm consumer
        x = _mk((M, N), 1.0, 8)
        x0 = x.clone()
        bias, g, bb = _mk((N,), 0.5, 9), _mk((N,), 1.0, 10), _mk((N,), 1.0, 11)
        y = torch.empty(M, N, device="cuda")
        lib.residual_layernorm(x, M, N, part, nz, M * N, bias, g, bb, out_f32=y)
        xr = x0 + bias + want
        assert (x - xr).abs().max().item() < 2e-3 * xr.abs().max().item()
        assert (y - F.layer_norm(xr, (N,), g, bb, 1e-5)).abs().max().item() < 5e-3
    err = (got - want).abs().max().item() / want.abs().max().item()
    report("gemm skinny M=%d N=%d K=%d tile=%d splitk=%d" % (M, N, K, tile_n, splitk), err)
    assert err < 2e-3


@pytest.mark.parametrize("M,N,K,tile_n,cluster,splitk,taps,batch", [
    (256, 3072, 1024, 32, 4, 1, 1, 1), (256, 1024, 4096, 32, 4, 4, 1, 1), (256, 4096, 1024, 64, 2, 1, 1, 1),
    (1872, 1024, 1024, 128, 4, 1, 3, 2), (300, 512, 128, 128, 2, 1, 1, 1), (77, 256, 256, 64, 4, 1, 3, 2)])
def test_gemm_cluster_multicast(M, N, K, tile_n, cluster, splitk, taps, batch):
    """Thread-block clusters along N with the activation tile multicast by TMA (gemm_mc.cuh)."""
    from tortoise_tts_b200 import lib
    A = _mk((batch, M, K), 1.0, 15).to(torch.bfloat16)
    W = _mk((N, taps, K), (K * taps) ** -0.5, 16).to(torch.bfloat16)
    a, w = A.float().cpu(), W.float().cpu()
    want = torch.zeros(batch, M, N)
    pad = (taps - 1) // 2
    for tap in range(taps):
        sh = tap - pad
        lo, hi = max(0, -sh), min(M, M - sh)
        want[:, lo:hi] += a[:, lo + sh:hi + sh] @ w[:, tap].t()
    want = want.cuda()
    if splitk == 1:
        b = _mk((N,), 0.5, 17)
        out = torch.full((batch, M, N), float("nan"), device="cuda")
        lib.gemm(A, W.reshape(N, taps * K), M=M, N=N, K=K, taps=taps, pad=pad, batch=batch, bias=b, out_f32=out,
                 a_bstride=M * K, outf_bstride=M * N, tile_n=tile_n, cluster=cluster)
        got = out - b
    else:
        kb = K // 64
        per = (kb + splitk - 1) // splitk
        nz = (kb + per - 1) // per
        part = torch.full((nz, M, N), float("nan"), device="cuda")
        lib.gemm(A, W.reshape(N, K), M=M, N=N, K=K, out_f32=part, outf_bstride=M * N, tile_n=tile_n, splitk=splitk,
                 cluster=cluster)
        got = part.sum(dim=0).unsqueeze(0)
    torch.cuda.synchronize()
    err = (got - want).abs().max().item() / want.abs().max().item()
    report("gemm cluster M=%d N=%d K=%d tile=%d cl=%d splitk=%d taps=%d" % (M, N, K, tile_n, cluster, splitk, taps), err)
    assert err < 2e-3


@pytest.mark.parametrize("case", [CASES[3], CASES[8], CASES[10]], ids=["tails", "conv3", "geglu"])
def test_gemm_simt_checker(case):
    y, of, ob = _run(force_ref=True, **case)
    scale = y.abs().max().item()
    got = of if of is not None else ob.float()
    err = (got - y).abs().max().item()
    report("gemm_ref %s" % case, err / scale)
    assert err / scale < 1e-2


EXPERIMENTAL = [
    dict(M=1872, N=1024, K=1024, taps=3, batch=2, residual=True, tile_n=128, variant=5),   # two TMA issuer threads
]


@pytest.mark.skipif(__import__("os").environ.get("TTB_TEST_EXPERIMENTAL") != "1",
                    reason="GEMM variant 5 (two TMA issuers) is not on the product path: opt in with TTB_TEST_EXPERIMENTAL=1")
@pytest.mark.parametrize("case", EXPERIMENTAL, ids=[str(i) for i in range(len(EXPERIMENTAL))])
def test_gemm_experimental_variants(case):
    y, of, ob = _run(**case)
    scale = y.abs().max().item()
    if of is not None:
        assert (of - y).abs().max().item() / scale < 2e-3
    if ob is not None:
        assert (ob.float() - y).abs().max().item() / scale < 1e-2
