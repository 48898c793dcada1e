"""GPU: the one-kernel GPT-2 decode step (csrc/ar_step.cu, ttb_ar_decode_step) phase by phase against fp32 torch on
the same inputs, at the production shapes of BASELINE configs[2]/[3] (B = 256 and 32 candidates, H = 16, P = 174), and the
whole step against the per-op path of round 1 and the CPU oracle.

Tolerances: GEMM operands are bf16 (weights and activations), accumulation / residual stream / LayerNorm / softmax are
fp32; outputs stored as bf16 carry 2^-9 relative rounding. Bounds are stated per check.
"""
import pytest
import torch
import torch.nn.functional as F

from gpu_util import report

pytestmark = pytest.mark.gpu

PH_EMBED, PH_QKV, PH_ATTN, PH_PROJ, PH_LN2, PH_FC, PH_PROJ2, PH_LN1, PH_HEAD = (1 << i for i in range(9))


def _rel(a, b):
    return (a.float() - b.float()).abs().max().item() / max(b.float().abs().max().item(), 1e-6)


def _mk(B, D, H, L, V, P, Nmax, step, seed=0, pos_mode=1, attn_compact=False):
    """Random weights / buffers for a stand-alone ArStep. Returns (handle, dict of tensors)."""
    from tortoise_tts_b200 import lib
    dev = "cuda"
    g = torch.Generator(device=dev)
    g.manual_seed(seed)

    def rn(*s, scale=1.0):
        return torch.randn(*s, generator=g, device=dev) * scale
    layers = []
    for _ in range(L):
        layers.append(dict(
            ln1_g=1 + rn(D, scale=0.1), ln1_b=rn(D, scale=0.1), ln2_g=1 + rn(D, scale=0.1), ln2_b=rn(D, scale=0.1),
            wqkv=rn(3 * D, D, scale=0.03).to(torch.bfloat16), bqkv=rn(3 * D, scale=0.1),
            wproj=rn(D, D, scale=0.03).to(torch.bfloat16), bproj=rn(D, scale=0.1),
            wfc=rn(4 * D, D, scale=0.03).to(torch.bfloat16), bfc=rn(4 * D, scale=0.1),
            wproj2=rn(D, 4 * D, scale=0.02).to(torch.bfloat16), bproj2=rn(D, scale=0.1)))
    t = dict(layers=layers,
             w_head=rn(V, D, scale=0.03).to(torch.bfloat16), b_head=rn(V, scale=0.1),
             lnf_g=1 + rn(D, scale=0.1), lnf_b=rn(D, scale=0.1), fn_g=1 + rn(D, scale=0.1), fn_b=rn(D, scale=0.1),
             mel_emb=rn(V, D, scale=0.05), mel_pos=rn(Nmax + 8, D, scale=0.05),
             codes=torch.randint(0, V - 2, (B, Nmax), generator=g, device=dev, dtype=torch.int32),
             state=torch.zeros(64, dtype=torch.int32, device=dev),
             x=rn(B, D), a=rn(B, D).to(torch.bfloat16), qkv=rn(B, 3 * D).to(torch.bfloat16),
             o=rn(B, D).to(torch.bfloat16), h=rn(B, 4 * D).to(torch.bfloat16), hn=rn(B, D).to(torch.bfloat16),
             logits=torch.zeros(B, V, device=dev),
             prefix_kv=rn(L, H, P, 2, 64).to(torch.bfloat16), cand_kv=rn(L, B, H, Nmax, 2, 64).to(torch.bfloat16))
    t["state"][0] = step
    hd = lib.ArStep(B=B, D=D, H=H, L=L, V=V, P=P, Nmax=Nmax, pos_mode=pos_mode, ld_codes=Nmax, attn_compact=attn_compact, **t)
    return hd, t


def _check_flag(t):
    torch.cuda.synchronize()
    assert int(t["state"][2].item()) == 0, "ar_step_kernel reported an internal time-out (code %d)" % int(t["state"][2])


def _mm(a_bf16, w_bf16, bias=None):
    y = a_bf16.float() @ w_bf16.float().t()
    return y if bias is None else y + bias


SHAPES = [  # B, D, H, V, P
    (256, 1024, 16, 8194, 174),      # configs[2]: all 256 candidates on one GPU
    (32, 1024, 16, 8194, 174),       # configs[3]: 32 candidates per GPU
    (96, 1024, 16, 8194, 44),        # preset 'fast', 10-word prompt
    (5, 128, 2, 300, 13),            # reduced config, ragged batch
]


@pytest.mark.parametrize("B,D,H,V,P", SHAPES)
def test_step_gemm_and_norm_phases(B, D, H, V, P):
    """Every non-attention phase of a layer, one at a time, against fp32 torch on identical bf16 operands."""
    L, Nmax, step = 2, 24, 3
    hd, t = _mk(B, D, H, L, V, P, Nmax, step, seed=B)
    lw = t["layers"][1]
    # --- embed + ln_1 of layer 0 (phase 0)
    hd.step(phase_mask=PH_EMBED, layer_begin=0, layer_end=1)
    _check_flag(t)
    tok = t["codes"][:, step - 1].long()
    x_ref = t["mel_emb"][tok] + t["mel_pos"][step + 1]
    assert torch.equal(t["x"], x_ref)
    a_ref = F.layer_norm(x_ref, (D,), t["layers"][0]["ln1_g"], t["layers"][0]["ln1_b"], 1e-5)
    r = _rel(t["a"], a_ref)
    report("ar_step embed+ln1 B=%d" % B, r)
    assert r < 6e-3                                   # bf16 store
    # --- c_attn of layer 1
    a_in = t["a"].clone()
    hd.step(phase_mask=PH_QKV, layer_begin=1, layer_end=2)
    _check_flag(t)
    r = _rel(t["qkv"], _mm(a_in, lw["wqkv"], lw["bqkv"]))
    report("ar_step c_attn B=%d" % B, r)
    assert r < 6e-3
    # --- c_proj (split-K partials) + residual + ln_2
    o_in, x_in = t["o"].clone(), t["x"].clone()
    hd.step(phase_mask=PH_PROJ | PH_LN2, layer_begin=1, layer_end=2)
    _check_flag(t)
    x_ref = x_in + _mm(o_in, lw["wproj"], lw["bproj"])
    r = _rel(t["x"], x_ref)
    report("ar_step c_proj+residual B=%d" % B, r)
    assert r < 1e-4                                   # fp32 accumulation order only
    r = _rel(t["a"], F.layer_norm(x_ref, (D,), lw["ln2_g"], lw["ln2_b"], 1e-5))
    assert r < 6e-3
    # --- c_fc + gelu_new
    a_in = t["a"].clone()
    hd.step(phase_mask=PH_FC, layer_begin=1, layer_end=2)
    _check_flag(t)
    r = _rel(t["h"], F.gelu(_mm(a_in, lw["wfc"], lw["bfc"]), approximate="tanh"))
    report("ar_step c_fc+gelu B=%d" % B, r)
    assert r < 8e-3
    # --- mlp.c_proj + residual + final norms (last layer -> ln_f -> final_norm -> hn)
    h_in, x_in = t["h"].clone(), t["x"].clone()
    hd.step(phase_mask=PH_PROJ2 | PH_LN1, layer_begin=1, layer_end=2)
    _check_flag(t)
    x_ref = x_in + _mm(h_in, lw["wproj2"], lw["bproj2"])
    r = _rel(t["x"], x_ref)
    report("ar_step mlp.c_proj+residual B=%d" % B, r)
    assert r < 1e-4
    hn_ref = F.layer_norm(F.layer_norm(x_ref, (D,), t["lnf_g"], t["lnf_b"], 1e-5), (D,), t["fn_g"], t["fn_b"], 1e-5)
    assert _rel(t["hn"], hn_ref) < 6e-3
    # ... and, for a non-final layer, the next layer's ln_1 into `a`
    x_in = t["x"].clone()
    hd.step(phase_mask=PH_PROJ2 | PH_LN1, layer_begin=0, layer_end=1)
    _check_flag(t)
    l0 = t["layers"][0]
    x_ref = x_in + _mm(h_in, l0["wproj2"], l0["bproj2"])
    assert _rel(t["x"], x_ref) < 1e-4
    assert _rel(t["a"], F.layer_norm(x_ref, (D,), lw["ln1_g"], lw["ln1_b"], 1e-5)) < 6e-3
    # --- mel_head
    hn_in = t["hn"].clone()
    hd.step(phase_mask=PH_HEAD, layer_begin=0, layer_end=0 + 1)
    _check_flag(t)
    r = _rel(t["logits"], _mm(hn_in, t["w_head"], t["b_head"]))
    report("ar_step mel_head B=%d" % B, r)
    assert r < 1e-4


@pytest.mark.parametrize("B,H,P", [(256, 16, 174), (32, 16, 174), (64, 16, 352), (7, 2, 13)])
@pytest.mark.parametrize("nc", [1, 7, 8, 9, 16, 17, 33, 215, 429])
@pytest.mark.parametrize("impl", ["mma", "simt"])
def test_step_attention_phase(B, H, P, nc, impl):
    """Decode attention over [shared prompt prefix | own KV | new token] + the KV append, at `nc` candidate entries
    (incl. the new one): all chunk-boundary cases of the 16-position ring and the production context lengths. `impl` is
    how the candidate's own cache is read: "mma" = the attention phase of the one-kernel step (TMA tiles, mma.sync);
    "simt" = the per-op decode attention (ttb_ar_decode_attention: SIMT stream over the own cache, prompt part on the
    tensor cores, merge) on the same inputs, with K and V in separate caches as that path keeps them."""
    from tortoise_tts_b200 import lib
    D, L, V, Nmax = H * 64, 2, 300, 430
    step = nc                                         # slot = step - 1 = nc - 1 old entries, + the new one
    hd, t = _mk(B, D, H, L, V, P, Nmax, step, seed=nc + B)
    layer = 1
    qkv = t["qkv"].clone()
    kv_before = t["cand_kv"].clone()
    if impl == "mma":
        hd.step(phase_mask=PH_ATTN, layer_begin=layer, layer_end=layer + 1)
        _check_flag(t)
        kv, o = t["cand_kv"], t["o"]
    else:
        ck_all, cv_all = kv_before[..., 0, :].contiguous(), kv_before[..., 1, :].contiguous()     # [L][B][H][Nmax][64]
        pk_l, pv_l = t["prefix_kv"][layer, :, :, 0].contiguous(), t["prefix_kv"][layer, :, :, 1].contiguous()
        o = torch.empty_like(t["o"])
        lib.ar_decode_attention(qkv, pk_l, pv_l, ck_all[layer], cv_all[layer], t["state"], B, H, P, Nmax, o,
                                torch.zeros(2, B, D, device="cuda"), torch.zeros(2, B, H, device="cuda"))
        _check_flag(t)
        kv = torch.stack([ck_all, cv_all], dim=-2)
    slot = step - 1
    # the append
    ck = kv[layer]
    assert torch.equal(ck[:, :, slot, 0], qkv[:, D:2 * D].reshape(B, H, 64))
    assert torch.equal(ck[:, :, slot, 1], qkv[:, 2 * D:].reshape(B, H, 64))
    mask = torch.ones_like(kv_before, dtype=torch.bool)
    mask[layer, :, :, slot] = False
    assert torch.equal(kv[mask], kv_before[mask]), "attention wrote outside the new slot"
    q = qkv[:, :D].reshape(B, H, 1, 64).float() * 0.125
    pk = t["prefix_kv"][layer, :, :, 0].float().unsqueeze(0).expand(B, -1, -1, -1)
    pv = t["prefix_kv"][layer, :, :, 1].float().unsqueeze(0).expand(B, -1, -1, -1)
    K = torch.cat([pk, ck[:, :, :slot + 1, 0].float()], dim=2)
    Vv = torch.cat([pv, ck[:, :, :slot + 1, 1].float()], dim=2)
    want = (torch.softmax(q @ K.transpose(-1, -2), -1) @ Vv).reshape(B, D)
    r = _rel(o, want)
    report("ar_step attention %s B=%d P=%d nc=%d" % (impl, B, P, nc), r)
    # mma: the softmax weights are rounded to bf16 for the P V product, as in every flash-attention kernel: 2^-9
    # relative on each weight, averaged over the row. simt: the same in the prompt part, fp32 weights over the own cache
    assert r < (8e-3 if impl == "mma" else 6e-3)


@pytest.mark.parametrize("B", [256, 32, 3])
def test_step_matches_per_op_path_and_is_deterministic(B):
    """Whole decode loop (full width, 2 layers): logits the sampler sees with the fused step vs the round-1 per-op path,
    same uniforms; graph replay == eager, bit for bit."""
    import os
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_all
    from tortoise_tts_b200 import ar_engine
    cfg = ModelConfig.medium()
    sd = synth_all(cfg, seed=1, suppress_stop=True)["autoregressive"]
    torch.manual_seed(0)
    text = torch.randint(1, 255, (169,)).tolist() + [0]
    cond = torch.randn(1, cfg.ar_dim)
    N = 20
    u = torch.rand(B, N)
    runs = {}
    for mode in ("fused", "mixed", "perop"):
        ar_engine.AREngine.MODE = mode
        eng = ar_engine.AREngine(sd, cfg)
        tr = []
        codes = eng.generate(cond, text, B, N, uniforms=u, trace_logits=tr).cpu()
        assert eng._dec["mode"] == mode
        runs[mode] = (codes, torch.stack([x.cpu() for x in tr], 1))
        if mode != "perop":
            codes_g = eng.generate(cond, text, B, N, uniforms=u, use_graph=True).cpu()
            assert torch.equal(codes_g, codes), "CUDA-graph replay of the %s step differs from eager" % mode
            codes_g2 = eng.generate(cond, text, B, N, uniforms=u, use_graph=True).cpu()
            assert torch.equal(codes_g2, codes)
        del eng
    ar_engine.AREngine.MODE = os.environ.get("TTB_AR_MODE", "auto")
    # Compare the logits on the common prefix of identical tokens (after the first nucleus-boundary flip the two runs
    # decode different sequences). Scale = the live logits (the synthetic checkpoint pins the stop / start logits at -1e4,
    # which would swamp a max-normalised error). The two paths round to bf16 at different points (split-K partial order,
    # fp32 vs bf16 softmax weights in the prompt part of the attention), so they agree to bf16 noise, not bit for bit.
    c0, l0 = runs["perop"]
    live = l0[0, 0].abs() < 1e3
    scale = l0[..., live].abs().max().item()
    for mode in ("fused", "mixed"):
        c1, l1 = runs[mode]
        worst = 0.0
        for b in range(B):
            same = (c1[b] == c0[b]).long().cumprod(0)
            n_cmp = min(N, int(same.sum()) + 1)
            worst = max(worst, (l1[b, :n_cmp][:, live] - l0[b, :n_cmp][:, live]).abs().max().item() / scale)
        report("ar_step %s vs per-op logits B=%d (rel. to live-logit scale %.1f)" % (mode, B, scale), worst)
        assert worst < 0.02
        report("ar_step %s vs per-op token agreement B=%d" % (mode, B), (c1 == c0).float().mean().item())


def test_step_full_depth_vs_oracle():
    """30 layers, full width, teacher-forced through the KV-cached fused decode loop vs the CPU oracle (fp32)."""
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_autoregressive
    from tortoise_tts_b200.ar_engine import AREngine
    from oracle import ar
    cfg = ModelConfig.full()
    sd = synth_autoregressive(cfg, 2, True)
    torch.manual_seed(0)
    text = torch.randint(1, 255, (20,)).tolist() + [0]
    cond = torch.randn(1, cfg.ar_dim)
    B, N = 2, 6
    u = torch.rand(B, N)
    eng = AREngine(sd, cfg)
    tr = []
    codes = eng.generate(cond, text, B, N, uniforms=u, trace_logits=tr).cpu().long()
    seen = torch.stack([x.cpu() for x in tr], 1)
    with torch.no_grad():
        want = ar.teacher_forced_logits(sd, cfg, cond, text, codes[:, :-1], "ref_kv_quirk")
    r = _rel(seen, want)
    report("ar_step full-depth decode logits vs oracle", r)
    assert r < 0.03


@pytest.mark.parametrize("B", [256, 128])
def test_two_chains_match_one_chain(B):
    """TTB_AR_CHAINS=2: the candidates decoded as two half-batches on two streams inside one (captured) step, with the
    attention in compact CTAs (`ar_attn_compact_kernel`, TtbArStepArgs.attn_compact). Every kernel of the step is
    row-independent, so codes and the logits the sampler sees must equal the one-chain run BIT FOR BIT, eager and as a
    graph replay (full width, 2 layers, prompt 174)."""
    import os
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_all
    from tortoise_tts_b200 import ar_engine
    cfg = ModelConfig.medium()
    sd = synth_all(cfg, seed=1, suppress_stop=True)["autoregressive"]
    torch.manual_seed(0)
    text = torch.randint(1, 255, (169,)).tolist() + [0]
    cond = torch.randn(1, cfg.ar_dim)
    N = 24
    u = torch.rand(B, N)
    E = ar_engine.AREngine
    saved = (E.MODE, E.CHAINS, E.CHAINS_MIN_B)
    runs = {}
    # one warp per (candidate, head) stream in both runs: with fewer candidates per CTA the planner would otherwise split
    # a stream over a team of warps, whose merge rounds differently (still correct, no longer bit-identical)
    os.environ["TTB_AR_STEP_TEAM"] = "1"
    try:
        E.MODE, E.CHAINS_MIN_B = "mixed", 64
        for nch in (1, 2):
            E.CHAINS = nch
            eng = E(sd, cfg)
            tr = []
            codes = eng.generate(cond, text, B, N, uniforms=u, trace_logits=tr).cpu()
            assert len(eng._dec["chains"]) == nch and bool(eng._dec["chains"][0]["compact"]) == (nch == 2)
            codes_g = eng.generate(cond, text, B, N, uniforms=u, use_graph=True).cpu()
            codes_g2 = eng.generate(cond, text, B, N, uniforms=u, use_graph=True).cpu()
            assert torch.equal(codes_g, codes) and torch.equal(codes_g2, codes), "graph replay differs (chains=%d)" % nch
            runs[nch] = (codes, torch.stack([x.cpu() for x in tr], 1))
            del eng
    finally:
        E.MODE, E.CHAINS, E.CHAINS_MIN_B = saved
        os.environ.pop("TTB_AR_STEP_TEAM", None)
    assert torch.equal(runs[1][0], runs[2][0])
    d = (runs[1][1] - runs[2][1]).abs().max().item()
    report("two decode chains vs one: max |logit difference| B=%d" % B, d)
    assert d == 0.0
