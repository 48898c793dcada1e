"""GPU: individual kernels behind the C-ABI against PyTorch fp32 / the oracle on the same inputs."""

import pytest
import torch
import torch.nn.functional as F

from gpu_util import report

pytestmark = pytest.mark.gpu


def test_device_ok():
    """The library accepts the device it is compiled for (compute capability 9.0)."""
    from tortoise_tts_b200 import lib
    torch.cuda.init()
    assert torch.cuda.get_device_capability() == (9, 0)
    assert lib.load().ttb_device_ok() == 1


def test_layernorm_single_and_chained():
    from tortoise_tts_b200 import lib
    torch.manual_seed(0)
    for D in (128, 1024):
        x = torch.randn(37, D, device="cuda") * 3 + 1
        g1, b1, g2, b2 = (torch.randn(D, device="cuda") for _ in range(4))
        of = torch.empty_like(x)
        lib.layernorm(x, 37, D, g1, b1, out_f32=of)
        want = F.layer_norm(x, (D,), g1, b1, 1e-5)
        assert (of - want).abs().max().item() < 1e-4
        ob = torch.empty(37, D, device="cuda", dtype=torch.bfloat16)
        lib.layernorm(x, 37, D, g1, b1, g2, b2, out_bf16=ob, out_f32=of)
        want = F.layer_norm(want, (D,), g2, b2, 1e-5)
        assert (of - want).abs().max().item() < 2e-4
        assert (ob.float() - want).abs().max().item() < 0.05


def test_rmsnorm():
    from tortoise_tts_b200 import lib
    from oracle.clvp import _rmsnorm
    torch.manual_seed(1)
    x = torch.randn(50, 768, device="cuda") * 2
    g = torch.randn(768, device="cuda")
    ob = torch.empty(50, 768, device="cuda", dtype=torch.bfloat16)
    lib.rmsnorm(x, 50, 768, g, ob)
    want = _rmsnorm(x.cpu(), g.cpu())
    assert (ob.float().cpu() - want).abs().max().item() < 0.05


@pytest.mark.parametrize("C,groups,S", [(128, 32, 45), (1024, 32, 374), (1024, 32, 1872), (96, 8, 33)])
def test_groupnorm_fused(C, groups, S):
    from tortoise_tts_b200 import lib
    torch.manual_seed(2)
    B = 2
    x = torch.randn(B, S, C, device="cuda") * 2 + 0.5
    gamma, beta = torch.randn(C, device="cuda"), torch.randn(C, device="cuda")
    ss = torch.randn(3, 2 * C, device="cuda") * 0.3
    row = torch.tensor([2], dtype=torch.int32, device="cuda")
    part = lib.groupnorm_scratch(B, groups, "cuda")
    of = torch.empty(B, S, C, device="cuda")
    ob = torch.empty(B, S, C, device="cuda", dtype=torch.bfloat16)
    lib.groupnorm(x, B, S, C, groups, gamma, beta, part, scale_shift=ss, ss_row=row, ss_row_stride=2 * C, silu=True,
                  out_bf16=ob, ldo=C, out_f32=of, ldof=C)
    want = F.group_norm(x.transpose(1, 2), groups, gamma, beta, 1e-5)
    want = want * (1 + ss[2, :C, None]) + ss[2, C:, None]
    want = F.silu(want).transpose(1, 2)
    err = (of - want).abs().max().item()
    report("groupnorm C=%d S=%d" % (C, S), err)
    assert err < 1e-3
    assert (ob.float() - want).abs().max().item() < 0.06
    # the same scratch serves later calls with another batch size (the denoiser's code_norm runs at B=1) and repeats
    for _ in range(2):
        of1 = torch.empty(1, S, C, device="cuda")
        lib.groupnorm(x[1:].contiguous(), 1, S, C, groups, gamma, beta, part, out_f32=of1, ldof=C)
        want1 = F.group_norm(x[1:].transpose(1, 2), groups, gamma, beta, 1e-5).transpose(1, 2)
        assert (of1 - want1).abs().max().item() < 1e-3
        lib.groupnorm(x, B, S, C, groups, gamma, beta, part, scale_shift=ss, ss_row=row, ss_row_stride=2 * C, silu=True,
                      out_f32=of, ldof=C)
        assert (of - want).abs().max().item() < 1e-3


@pytest.mark.parametrize("S,taps,residual,kw", [(1872, 3, True, {}), (1872, 1, False, {}), (43, 1, True, {}),
                                                 (500, 3, True, dict(variant=2)), (256, 1, False, dict(tile_n=64)),
                                                 (1000, 1, True, dict(cluster=2)), (2176, 3, True, {})])
def test_gemm_groupnorm_statistics_in_epilogue(S, taps, residual, kw):
    """TtbGemmArgs.gn_partials: the GEMM epilogue leaves (sum, sum of squares) per 32 x 32 output block and
    ttb_groupnorm_apply normalises from them; against F.group_norm of the GEMM's own fp32 output (GroupNorm32,
    arch_util.py:21-41) and against the two-pass ttb_groupnorm."""
    from tortoise_tts_b200 import lib
    torch.manual_seed(11)
    B, C, groups = 2, 1024, 32
    a = (torch.randn(B, S, C, device="cuda") * 0.5).to(torch.bfloat16)
    w = (torch.randn(C, taps * C, device="cuda") * 0.03).to(torch.bfloat16)
    bias = torch.randn(C, device="cuda")
    x = torch.randn(B, S, C, device="cuda") + 0.3
    part = lib.groupnorm_scratch(B, groups, "cuda")
    part.fill_(float("nan"))                       # every partial that is read must have been written by the GEMM
    out = x.clone() if residual else torch.empty_like(x)
    lib.gemm(a, w, M=S, N=C, K=C, taps=taps, pad=taps // 2, bias=bias, residual=out if residual else None, out_f32=out,
             batch=B, a_bstride=S * C, res_bstride=S * C, outf_bstride=S * C, gn_partials=part, gn_groups=groups, **kw)
    gamma, beta = torch.randn(C, device="cuda"), torch.randn(C, device="cuda")
    got = torch.empty(B, S, C, device="cuda")
    lib.groupnorm_apply(out, B, S, C, groups, gamma, beta, part, silu=True, out_f32=got, ldof=C)
    want = F.silu(F.group_norm(out.transpose(1, 2), groups, gamma, beta, 1e-5)).transpose(1, 2)
    err = (got - want).abs().max().item()
    report("gemm-epilogue groupnorm statistics S=%d taps=%d %s" % (S, taps, kw), err)
    assert err < 1e-3
    two = torch.empty(B, S, C, device="cuda")
    lib.groupnorm(out, B, S, C, groups, gamma, beta, lib.groupnorm_scratch(B, groups, "cuda"), silu=True, out_f32=two, ldof=C)
    assert (got - two).abs().max().item() < 1e-3


@pytest.mark.parametrize("T,C,N,k,dil", [(1000, 64, 64, 3, 3), (517, 256, 256, 11, 5), (2000, 32, 32, 7, 1), (300, 128, 1, 7, 1)])
def test_gemm_dilated_taps_split_operands(T, C, N, k, dil):
    """Dilated Conv1d as ONE GEMM (TtbGemmArgs.tap_dilation) on error-compensated operands (ttb_act_split_cast triple
    [hi | lo | hi] x [Wh | Wh | Wl]) with leaky_relu on the input and tanh on the output, against F.conv1d in fp32
    (hifigan_decoder.py:92-95: xt = conv(leaky_relu(x)))."""
    from tortoise_tts_b200 import lib
    from tortoise_tts_b200.hifigan_engine import _kt, _pack_conv
    torch.manual_seed(13)
    x = torch.randn(T, C, device="cuda")
    w = torch.randn(N, C, k) * (1.0 / (C * k) ** 0.5)
    b = torch.randn(N, device="cuda") * 0.1
    a = torch.empty(T, _kt(C), dtype=torch.bfloat16, device="cuda")
    lib.act_split_cast(x, T, C, a, _kt(C), slope=0.1)
    out = torch.empty(T, N, device="cuda")
    lib.gemm(a, _pack_conv(w, "cuda"), M=T, N=N, K=_kt(C), taps=k, pad=dil * (k - 1) // 2, tap_dilation=dil, bias=b,
             out_f32=out, act=lib.ACT_TANH, tile_n=32 if N <= 32 else 0)
    want = torch.tanh(F.conv1d(F.leaky_relu(x, 0.1).t().unsqueeze(0), w.cuda(), b, dilation=dil,
                               padding=dil * (k - 1) // 2))[0].t()
    err = (out - want).abs().max().item()
    report("dilated conv GEMM, split operands T=%d C=%d N=%d k=%d d=%d" % (T, C, N, k, dil), err)
    assert err < 2e-4


def test_interp_linear():
    """F.interpolate(mode='linear') with an explicit scale factor, twice, as HifiganGenerator.inference does."""
    from tortoise_tts_b200 import lib
    torch.manual_seed(14)
    L, C = 57, 64
    x = torch.randn(L, C, device="cuda")
    T1 = int(L * 4.0)
    T = int(T1 * (24000 / 22050))
    u1 = torch.empty(T1, C, device="cuda")
    lib.interp_linear(x, L, C, 0.25, T1, u1)
    u2 = torch.empty(T, C, device="cuda")
    lib.interp_linear(u1, T1, C, 22050.0 / 24000.0, T, u2)
    w1 = F.interpolate(x.t().unsqueeze(0), scale_factor=[4.0], mode="linear")
    w2 = F.interpolate(w1, scale_factor=[24000 / 22050], mode="linear")
    assert w2.shape[-1] == T
    assert (u1 - w1[0].t()).abs().max().item() < 1e-5
    assert (u2 - w2[0].t()).abs().max().item() < 1e-5


@pytest.mark.parametrize("T,H,nseq,causal,use_bias", [(45, 2, 2, False, True), (174, 16, 1, True, False),
                                                      (374, 16, 2, False, True), (130, 12, 3, False, False),
                                                      (64, 2, 1, False, False), (128, 2, 2, True, True),
                                                      (1872, 16, 2, False, True), (676, 16, 1, True, False),
                                                      (1872, 16, 2, False, "t5"), (500, 4, 1, True, "t5"),
                                                      (300, 4, 2, False, "big"), (256, 2, 1, True, True),
                                                      (257, 3, 1, False, "t5"), (430, 12, 2, False, False),
                                                      (193, 2, 2, True, False), (1000, 2, 1, True, "big")])
def test_attention(T, H, nseq, causal, use_bias):
    from tortoise_tts_b200 import lib
    from tortoise_tts_b200.diffusion_engine import _rel_pos_table
    torch.manual_seed(3)
    D = H * 64
    # "big": scores spanning > 2^8 so that the lazy O rescale is exercised
    qkv = (torch.randn(nseq * T, 3 * D, device="cuda") * (4.0 if use_bias == "big" else 1.0)).to(torch.bfloat16)
    sat = 0
    if use_bias == "t5":      # saturated T5 relative-position table (fast-tile path of the flash kernel)
        bias, sat = _rel_pos_table(torch.randn(32, H, device="cuda"), T, 8.0), 64
    elif use_bias is True:
        bias = torch.randn(H, 2 * T - 1, device="cuda")
    else:
        bias, use_bias = None, False
    out = torch.empty(nseq * T, D, device="cuda", dtype=torch.bfloat16)
    lib.attention(qkv, out, nseq=nseq, T=T, H=H, ld=3 * D, ldo=D, k_off=D, v_off=2 * D, scale=0.125, causal=causal,
                  bias=bias, bias_sat=sat)
    q, k, v = (t.float().view(nseq, T, H, 64).transpose(1, 2) for t in qkv.split(D, dim=1))
    w = (q @ k.transpose(-1, -2)) * 0.125
    if use_bias:
        i = torch.arange(T, device="cuda")
        idx = i[None, :] - i[:, None] + T - 1
        w = w + bias[:, idx].unsqueeze(0)
    if causal:
        w = w.masked_fill(~torch.ones(T, T, dtype=torch.bool, device="cuda").tril(), float("-inf"))
    want = (torch.softmax(w, -1) @ v).transpose(1, 2).reshape(nseq * T, D)
    # outputs are bf16: tolerance relative to the output scale (|v| reaches ~15 in the "big" case)
    err = (out.float() - want).abs().max().item() / max(1.0, want.abs().max().item() / 4.0)
    report("attention T=%d causal=%d bias=%s" % (T, causal, use_bias), err)
    assert err < 0.03


def test_sampler_matches_oracle():
    """Fused sampler vs the oracle's closed form of the HF processor chain on identical logits / uniforms."""
    from tortoise_tts_b200 import lib
    from oracle import ar
    torch.manual_seed(4)
    B, V, N = 24, 8194, 3
    logits = (torch.randn(B, V) * 3).cuda()
    u = torch.rand(B, N).cuda()
    seen = torch.zeros(B, (V + 31) // 32, dtype=torch.int32, device="cuda")
    seen[:, 0] = 2
    seen[:, 256] |= 1
    prev = [[1, 8192] + torch.randint(0, 8192, (15,)).tolist() for _ in range(B)]
    for b in range(B):
        for t in prev[b][2:]:
            seen[b, t // 32] |= (1 << (t % 32)) if t % 32 < 31 else -(1 << 31)
    codes = torch.full((B, N), -1, dtype=torch.int32, device="cuda")
    fin = torch.zeros(B, dtype=torch.int32, device="cuda")
    fin[3] = 1
    state = torch.zeros(64, dtype=torch.int32, device="cuda")
    lib.ar_sample(logits, V, V, B, u, N, seen, codes, N, fin, state, 0.8, 50, 0.8, 2.0, 8193, advance=True)
    torch.cuda.synchronize()
    assert int(state[0]) == 1 and int(state[1]) == 0
    mism = 0
    for b in range(B):
        if b == 3:
            assert int(codes[b, 0]) == 8193
            continue
        tok, kept, kp = ar.sample_step(logits[b].cpu(), prev[b], float(u[b, 0]))
        if tok != int(codes[b, 0]):
            mism += 1
            assert int(codes[b, 0]) in kept.tolist()   # boundary effects only
    assert mism <= 1
    # second step: repetition penalty must now see the token just sampled
    w, bit = divmod(int(codes[0, 0]), 32)
    assert (int(seen[0, w]) >> bit) & 1


def test_sampler_distribution():
    """chi-square of 4000 draws against the oracle's kept probabilities."""
    from tortoise_tts_b200 import lib
    from oracle import ar
    torch.manual_seed(5)
    V, B = 8194, 4000
    row = torch.randn(1, V) * 3
    logits = row.cuda()
    u = torch.rand(B, 1).cuda()
    seen = torch.zeros(B, (V + 31) // 32, dtype=torch.int32, device="cuda")
    codes = torch.full((B, 1), -1, dtype=torch.int32, device="cuda")
    fin = torch.zeros(B, dtype=torch.int32, device="cuda")
    state = torch.zeros(64, dtype=torch.int32, device="cuda")
    lib.ar_sample(logits, 0, V, B, u, 1, seen, codes, 1, fin, state, 0.8, 50, 0.8, 2.0, 8193, advance=False)
    _, kept, kp = ar.sample_step(row[0], [], 0.5)
    counts = torch.bincount(codes[:, 0].long().cpu(), minlength=V)[kept]
    assert counts.sum().item() == B
    exp = kp * B
    chi2 = ((counts - exp) ** 2 / exp).sum().item()
    report("sampler chi2 (dof=%d)" % (len(kp) - 1), chi2)
    assert chi2 < 3 * len(kp) + 20


def test_fix_codes():
    from tortoise_tts_b200 import lib
    from oracle import ar
    rows = [[5, 6, 7, 8193, 8193, 8193, 8193, 8193, 8193, 8193, 8193, 8193, 8193, 8193, 8193, 8193],
            list(range(16)), [8193] + [3] * 15, [3] * 15 + [8193], [83] * 10 + [4] * 6]
    c = torch.tensor(rows, dtype=torch.int32, device="cuda")
    trim = torch.empty(len(rows), dtype=torch.int32, device="cuda")
    lib.ar_fix_codes(c, len(rows), 16, 8193, trim)
    for i, r in enumerate(rows):
        want = ar.fix_autoregressive_output(torch.tensor(r), 8193)
        assert c[i].cpu().tolist() == want.tolist()
        assert int(trim[i]) == ar.calm_trim_length(want)


def test_diffusion_step_kernel():
    """ttb_diffusion_step at the first, a middle and the last call, with and without classifier-free guidance. `parity`
    lays model_out out as the double-buffered peer-exchange area (parity_stride) of the two-GPU CFG pair, with the other
    slot holding garbage. The bf16 copy leaves columns C..ld_xb-1 alone, and the mel is written at the last call (i == 0)
    only."""
    from tortoise_tts_b200 import lib
    from tortoise_tts_b200.diffusion_engine import make_schedule
    torch.manual_seed(6)
    S, C, iters, ld_xb = 50, 100, 7, 128
    tmap, tables = make_schedule(iters)
    tb = torch.from_numpy(tables).cuda()
    n = S * 2 * C
    for cond_free, parity in ((True, False), (False, False), (True, True), (False, True)):
        for call in (0, 3, 6):
            i = iters - 1 - call
            mo = torch.randn(2, S, 2 * C, device="cuda")
            if parity:
                area = torch.full((2, 2 * n), float("nan"), device="cuda")
                area[call & 1] = mo.reshape(-1)
                model_out, stride = area, 2 * n
            else:
                model_out, stride = mo, 0
            x = torch.randn(S, C, device="cuda")
            x0 = x.clone()
            noise = torch.randn(iters, S, C, device="cuda")
            xb = torch.full((S, ld_xb), float("nan"), device="cuda", dtype=torch.bfloat16)
            step = torch.tensor([call], dtype=torch.int32, device="cuda")
            mel = torch.full((C, S), float("nan"), device="cuda")
            lib.diffusion_step(model_out, n, 2 * C, x, xb, ld_xb, noise, tb, step, S, C, iters, cond_free, 2.0, mel,
                               parity_stride=stride)
            eps, var = mo[0, :, :C], mo[0, :, C:]
            if cond_free:
                cfk = 2.0 * (1 - i / iters)
                eps = (1 + cfk) * eps - cfk * mo[1, :, :C]
            frac = (var + 1) / 2
            logvar = frac * tb[3, i] + (1 - frac) * tb[2, i]
            xs = (tb[0, i] * x0 - tb[1, i] * eps).clamp(-1, 1)
            mean = tb[4, i] * xs + tb[5, i] * x0
            want = mean + (0.0 if i == 0 else 1.0) * torch.exp(0.5 * logvar) * noise[call]
            assert (x - want).abs().max().item() < 1e-4
            assert torch.equal(xb[:, :C], x.to(torch.bfloat16))
            assert torch.isnan(xb[:, C:].float()).all()
            if i == 0:
                wm = ((want + 1) / 2) * (2.3143386840820312 + 11.512925148010254) - 11.512925148010254
                assert (mel - wm.t()).abs().max().item() < 1e-3
            else:
                assert torch.isnan(mel).all()


def test_vocoder_convs():
    from tortoise_tts_b200 import lib
    torch.manual_seed(7)
    # plain / dilated / reflect convs
    for (cin, cout, k, dil, reflect, L) in [(100, 64, 5, 1, False, 77), (32, 32, 3, 27, False, 600), (64, 32, 7, 1, True, 50),
                                            (32, 1, 7, 1, True, 333)]:
        x = torch.randn(cin, L, device="cuda")
        w = torch.randn(cout, cin, k, device="cuda") * (cin * k) ** -0.5
        b = torch.randn(cout, device="cuda")
        res = torch.randn(cout, L, device="cuda")
        out = torch.empty(cout, L, device="cuda")
        lib.voc_conv1d(x, cin, L, w, b, cout, k, out, dilation=dil, reflect=reflect, lrelu_in=0.2, lrelu_out=0.2,
                       residual=res)
        xi = F.leaky_relu(x, 0.2).unsqueeze(0)
        pad = dil * (k // 2)
        xi = F.pad(xi, (pad, pad), mode="reflect" if reflect else "constant")
        want = F.leaky_relu(F.conv1d(xi, w, b, dilation=dil), 0.2)[0] + res
        assert (out - want).abs().max().item() < 1e-4, (cin, cout, k, dil)
    # transposed conv
    for s, L in ((8, 40), (4, 123)):
        x = torch.randn(32, L, device="cuda")
        w = torch.randn(32, 32, 2 * s, device="cuda") * 0.1
        b = torch.randn(32, device="cuda")
        out = torch.empty(32, L * s, device="cuda")
        lib.voc_convt(x, 32, L, w, b, s, 0.2, out)
        want = F.conv_transpose1d(F.leaky_relu(x, 0.2).unsqueeze(0), w, b, stride=s, padding=s // 2 + s % 2,
                                  output_padding=s % 2)[0]
        assert (out - want).abs().max().item() < 1e-4, s


@pytest.mark.parametrize("hop,Fr", [(8, 21), (64, 9), (256, 5)])
def test_vocoder_lvc_gate(hop, Fr):
    from tortoise_tts_b200 import lib
    from oracle.vocoder import lvc
    torch.manual_seed(8)
    C, L = 32, hop * Fr
    y = torch.randn(C, L)
    K = torch.randn(C, 2 * C, 3, Fr) * 0.1          # reference layout [in, out, k, F]
    Bi = torch.randn(2 * C, Fr)
    x = torch.randn(C, L)
    o = lvc(y, K, Bi, hop)
    want = x + torch.sigmoid(o[:C]) * torch.tanh(o[C:])
    ldk = 4 * 6144 + 256
    kern = torch.zeros(Fr, ldk)
    layer = 2
    kern[:, layer * 6144:(layer + 1) * 6144] = K.permute(3, 0, 2, 1).reshape(Fr, -1)   # [F][i][k][oc]
    kern[:, 4 * 6144 + layer * 64: 4 * 6144 + (layer + 1) * 64] = Bi.t()
    kern = kern.cuda()
    xg = x.cuda()
    lib.voc_lvc_gate(y.cuda(), C, L, hop, kern, ldk, layer * 6144, kern, ldk, 4 * 6144 + layer * 64, xg)
    err = (xg.cpu() - want).abs().max().item()
    report("lvc_gate hop=%d" % hop, err)
    assert err < 1e-4


def test_misc_kernels():
    from tortoise_tts_b200 import lib
    from oracle import diffusion as od
    torch.manual_seed(9)
    t = torch.tensor([3979, 0, 20], dtype=torch.int32, device="cuda")
    out = torch.empty(3, 1024, device="cuda")
    lib.timestep_embedding(t, 3, 1024, out)
    want = od.timestep_embedding(t.cpu().long(), 1024)
    assert (out.cpu() - want).abs().max().item() < 2e-3   # fast-math sin/cos at arguments up to 4e3
    x = torch.randn(5, 256, device="cuda")
    W, b = torch.randn(300, 256, device="cuda") * 0.05, torch.randn(300, device="cuda")
    y = torch.empty(5, 300, device="cuda")
    lib.linear_small(x, 5, 256, W, b, 300, y, silu_in=True, silu_out=True)
    assert (y - F.silu(F.linear(F.silu(x), W, b))).abs().max().item() < 1e-4
    xi = torch.randn(10, 64, device="cuda")
    o = torch.empty(43, 64, device="cuda")
    lib.interp_nearest(xi, 10, 43, 64, out_f32=o, ldof=64)
    want = F.interpolate(xi.t().unsqueeze(0), size=43, mode="nearest")[0].t()
    assert torch.equal(o, want)
    a = torch.randn(100, 37, device="cuda")
    tr = torch.empty(37, 100, device="cuda")
    lib.transpose_f32(a, 100, 37, tr)
    assert torch.equal(tr, a.t())
    # CLVP rotary vs oracle
    from oracle.clvp import _rotary
    H, T = 2, 9
    qkv = torch.randn(2 * T, 3 * H * 64, device="cuda").to(torch.bfloat16)
    ref = qkv.float().cpu().view(2, T, 3 * H, 64)
    f = torch.einsum("i,j->ij", torch.arange(T).float(), 1.0 / (10000 ** (torch.arange(0, 32, 2).float() / 32)))
    fr = torch.cat((f, f), -1)[None, :, None, :]
    want = torch.cat((_rotary(ref[..., :32], fr), ref[..., 32:]), -1).reshape(2 * T, -1)
    lib.clvp_rotary(qkv, 2, T, H)
    assert (qkv.float().cpu() - want).abs().max().item() < 0.03
