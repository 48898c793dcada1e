"""GPU: prompt groups in the decode step (TtbArStepArgs.groups) and the batch decode behind TextToSpeech.tts_batch.

The attention phase with several prompt prefixes against fp32 torch; the grouped decode loop against generate() of each
utterance alone (bit for bit where the step is row-independent, to bf16 noise for the one-kernel step) and against the
CPU oracle at full depth; tts_batch against one tts() call per text."""
import os

import pytest
import torch

from gpu_util import report

pytestmark = pytest.mark.gpu

PH_ATTN = 4


def _rel(a, b):
    return (a.float() - b.float()).abs().max().item() / max(b.float().abs().max().item(), 1e-6)


def _grouped_step(sizes, Ps, H, L, Nmax, step, seed, attn_compact):
    """A stand-alone ArStep whose rows form len(sizes) prompt groups with their own random prefixes."""
    from tortoise_tts_b200 import lib
    dev = "cuda"
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    D, V, B = H * 64, 300, sum(sizes)

    def rn(*s, scale=1.0):
        return torch.randn(*s, generator=g, device=dev) * scale
    layers = [dict(ln1_g=1 + rn(D, scale=0.1), ln1_b=rn(D, scale=0.1), ln2_g=1 + rn(D, scale=0.1), ln2_b=rn(D, scale=0.1),
                   wqkv=rn(3 * D, D, scale=0.03).to(torch.bfloat16), bqkv=rn(3 * D, scale=0.1),
                   wproj=rn(D, D, scale=0.03).to(torch.bfloat16), bproj=rn(D, scale=0.1),
                   wfc=rn(4 * D, D, scale=0.03).to(torch.bfloat16), bfc=rn(4 * D, scale=0.1),
                   wproj2=rn(D, 4 * D, scale=0.02).to(torch.bfloat16), bproj2=rn(D, scale=0.1)) for _ in range(L)]
    prefixes = [rn(L, H, P, 2, 64).to(torch.bfloat16) for P in Ps]
    groups, b = [], 0
    for n, P, pkv in zip(sizes, Ps, prefixes):
        groups.append((b, b + n, P, pkv))
        b += n
    t = dict(layers=layers, w_head=rn(V, D, scale=0.03).to(torch.bfloat16), b_head=rn(V, scale=0.1),
             lnf_g=1 + rn(D, scale=0.1), lnf_b=rn(D, scale=0.1), fn_g=1 + rn(D, scale=0.1), fn_b=rn(D, scale=0.1),
             mel_emb=rn(V, D, scale=0.05), mel_pos=rn(Nmax + 8, D, scale=0.05),
             codes=torch.randint(0, V - 2, (B, Nmax), generator=g, device=dev, dtype=torch.int32),
             state=torch.zeros(64, dtype=torch.int32, device=dev),
             x=rn(B, D), a=rn(B, D).to(torch.bfloat16), qkv=rn(B, 3 * D).to(torch.bfloat16),
             o=rn(B, D).to(torch.bfloat16), h=rn(B, 4 * D).to(torch.bfloat16), hn=rn(B, D).to(torch.bfloat16),
             logits=torch.zeros(B, V, device=dev), prefix_kv=prefixes[0],
             cand_kv=rn(L, B, H, Nmax, 2, 64).to(torch.bfloat16))
    t["state"][0] = step
    hd = lib.ArStep(B=B, D=D, H=H, L=L, V=V, P=Ps[0], Nmax=Nmax, pos_mode=1, ld_codes=Nmax, attn_compact=attn_compact,
                    groups=groups, **t)
    return hd, t, groups


GROUPINGS = [  # group sizes, prompt lengths
    ([1, 5, 10], [13, 174, 352]),              # 16 rows, a group of one
    ([50, 1, 77], [352, 13, 174]),             # 128 rows, uneven
    ([37, 100, 119], [174, 352, 13]),          # 256 rows
]


@pytest.mark.parametrize("sizes,Ps", GROUPINGS)
@pytest.mark.parametrize("nc", [1, 17, 215])
@pytest.mark.parametrize("compact", [False, True])
def test_grouped_attention_phase(sizes, Ps, nc, compact):
    """The attention phase (debug_phase_mask = 4, one layer) with per-group prompt prefixes, against fp32 torch: every
    row attends to [its group's prefix | own KV | new token], and only the new slot of the cache is written."""
    H, L, Nmax, layer = 16, 2, 430, 1
    D = H * 64
    hd, t, groups = _grouped_step(sizes, Ps, H, L, Nmax, nc, seed=nc + sum(sizes), attn_compact=compact)
    qkv = t["qkv"].clone()
    kv_before = t["cand_kv"].clone()
    hd.step(phase_mask=PH_ATTN, layer_begin=layer, layer_end=layer + 1)
    torch.cuda.synchronize()
    assert int(t["state"][2].item()) == 0, "internal time-out in the attention phase"
    slot = nc - 1
    ck = t["cand_kv"][layer]
    B = sum(sizes)
    assert torch.equal(ck[:, :, slot, 0], qkv[:, D:2 * D].reshape(B, H, 64))
    assert torch.equal(ck[:, :, slot, 1], qkv[:, 2 * D:].reshape(B, H, 64))
    mask = torch.ones_like(kv_before, dtype=torch.bool)
    mask[layer, :, :, slot] = False
    assert torch.equal(t["cand_kv"][mask], kv_before[mask]), "attention wrote outside the new slot"
    worst = 0.0
    for b0, b1, P, pkv in groups:
        n = b1 - b0
        q = qkv[b0:b1, :D].reshape(n, H, 1, 64).float() * 0.125
        pk = pkv[layer, :, :, 0].float().unsqueeze(0).expand(n, -1, -1, -1)
        pv = pkv[layer, :, :, 1].float().unsqueeze(0).expand(n, -1, -1, -1)
        K = torch.cat([pk, ck[b0:b1, :, :slot + 1, 0].float()], dim=2)
        Vv = torch.cat([pv, ck[b0:b1, :, :slot + 1, 1].float()], dim=2)
        want = (torch.softmax(q @ K.transpose(-1, -2), -1) @ Vv).reshape(n, D)
        worst = max(worst, _rel(t["o"][b0:b1], want))
    report("grouped attention sizes=%s P=%s nc=%d compact=%d" % (sizes, Ps, nc, compact), worst)
    assert worst < 8e-3                        # the bound of test_step_attention_phase (bf16 softmax weights in P V)


def _engine_setup():
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_all
    cfg = ModelConfig.medium()
    sd = synth_all(cfg, seed=1, suppress_stop=True)["autoregressive"]
    torch.manual_seed(0)
    texts = [torch.randint(1, 255, (n,)).tolist() + [0] for n in (169, 40, 300)]    # P = 174, 45, 305
    return cfg, sd, texts, torch.randn(1, cfg.ar_dim)


@pytest.mark.parametrize("chains", [1, 2])
def test_grouped_decode_is_bit_identical_to_each_utterance_alone(chains):
    """TTB_AR_STEP_TEAM=1, mixed step: three utterances (128 rows; with two chains the middle group straddles the split)
    decoded as one batch give each group's rows the codes and logits of generate() of that utterance alone, bit for
    bit, eager and as a graph replay."""
    from tortoise_tts_b200 import ar_engine
    cfg, sd, texts, cond = _engine_setup()
    counts, N = [40, 50, 38], 24
    us = [torch.rand(n, N) for n in counts]
    E = ar_engine.AREngine
    saved = (E.MODE, E.CHAINS, E.CHAINS_MIN_B)
    os.environ["TTB_AR_STEP_TEAM"] = "1"
    try:
        E.MODE, E.CHAINS, E.CHAINS_MIN_B = "mixed", chains, 64
        eng = E(sd, cfg)
        tr = []
        got = eng.generate_grouped(cond, texts, counts, N, uniforms_list=us, trace_logits=tr)
        assert len(eng._dec["chains"]) == chains
        seen = torch.stack([x.cpu() for x in tr], 1)
        got_g = eng.generate_grouped(cond, texts, counts, N, uniforms_list=us, use_graph=True)
        for a, b in zip(got, got_g):
            assert torch.equal(a, b), "graph replay of the grouped step differs from eager"
        b0 = 0
        for u, n in enumerate(counts):
            tr1 = []
            want = eng.generate(cond, texts[u], n, N, uniforms=us[u], trace_logits=tr1)
            assert eng._dec["mode"] == "mixed"
            assert torch.equal(got[u].cpu(), want.cpu()), "codes of utterance %d differ" % u
            d = (seen[b0:b0 + n] - torch.stack([x.cpu() for x in tr1], 1)).abs().max().item()
            report("grouped vs alone, max |logit difference| chains=%d u=%d" % (chains, u), d)
            assert d == 0.0
            b0 += n
    finally:
        E.MODE, E.CHAINS, E.CHAINS_MIN_B = saved
        os.environ.pop("TTB_AR_STEP_TEAM", None)


def test_fused_grouped_step_matches_each_utterance_alone():
    """The one-kernel step with 3 groups of 4 / 5 / 7 rows against each utterance decoded alone by the same step: within
    bf16 noise of the live-logit scale on the common prefix of identical tokens; graph replay == eager."""
    from tortoise_tts_b200 import ar_engine
    cfg, sd, texts, cond = _engine_setup()
    counts, N = [4, 5, 7], 20
    us = [torch.rand(n, N) for n in counts]
    E = ar_engine.AREngine
    saved = E.MODE
    try:
        E.MODE = "fused"
        eng = E(sd, cfg)
        tr = []
        got = eng.generate_grouped(cond, texts, counts, N, uniforms_list=us, trace_logits=tr)
        assert eng._dec["mode"] == "fused"
        seen = torch.stack([x.cpu() for x in tr], 1)
        for _ in range(2):
            got_g = eng.generate_grouped(cond, texts, counts, N, uniforms_list=us, use_graph=True)
            for a, b in zip(got, got_g):
                assert torch.equal(a, b), "graph replay of the fused grouped step differs from eager"
        b0 = 0
        for u, n in enumerate(counts):
            tr1 = []
            want = eng.generate(cond, texts[u], n, N, uniforms=us[u], trace_logits=tr1).cpu()
            l0 = torch.stack([x.cpu() for x in tr1], 1)
            live = l0[0, 0].abs() < 1e3
            scale = l0[..., live].abs().max().item()
            worst = 0.0
            for r in range(n):
                same = (got[u][r].cpu() == want[r]).long().cumprod(0)
                n_cmp = min(N, int(same.sum()) + 1)
                worst = max(worst, (seen[b0 + r, :n_cmp][:, live] - l0[r, :n_cmp][:, live]).abs().max().item() / scale)
            report("fused grouped vs alone logits u=%d (rel. to live-logit scale %.1f)" % (u, scale), worst)
            assert worst < 0.02
            b0 += n
    finally:
        E.MODE = saved


def test_grouped_full_depth_vs_oracle():
    """30 layers, full width, two utterances with different prompts in one batch: the logits each group's rows see
    against the CPU oracle teacher-forced on that group's prompt and codes (fp32)."""
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_autoregressive
    from tortoise_tts_b200.ar_engine import AREngine
    from oracle import ar
    cfg = ModelConfig.full()
    sd = synth_autoregressive(cfg, 2, True)
    torch.manual_seed(0)
    texts = [torch.randint(1, 255, (20,)).tolist() + [0], torch.randint(1, 255, (57,)).tolist() + [0]]
    cond = torch.randn(1, cfg.ar_dim)
    counts, N = [2, 3], 6
    us = [torch.rand(n, N) for n in counts]
    eng = AREngine(sd, cfg)
    tr = []
    got = eng.generate_grouped(cond, texts, counts, N, uniforms_list=us, trace_logits=tr)
    seen = torch.stack([x.cpu() for x in tr], 1)
    b0 = 0
    for u, n in enumerate(counts):
        with torch.no_grad():
            want = ar.teacher_forced_logits(sd, cfg, cond, texts[u], got[u].cpu().long()[:, :-1], "ref_kv_quirk")
        r = _rel(seen[b0:b0 + n], want)
        report("grouped full-depth decode logits vs oracle u=%d" % u, r)
        assert r < 0.03
        b0 += n


def _facade():
    from tortoise_tts_b200.api import TextToSpeech
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_all
    cfg = ModelConfig.small()
    return TextToSpeech(state_dicts=synth_all(cfg, seed=0, suppress_stop=False), config=cfg, enable_redaction=False), cfg


def test_tts_batch_equals_tts_per_text():
    """TTB_AR_MODE=mixed with one warp per stream: tts_batch of five texts (the third with a prompt of 354 positions,
    decoded alone between two grouped batches) returns exactly the waveforms of one tts() call per text. With the default step: finite waveforms of
    the per-text lengths, and a second call replays the captured grouped step."""
    from tortoise_tts_b200 import ar_engine
    tts, cfg = _facade()
    torch.manual_seed(5)
    toks = [torch.randint(1, 255, (n,)).tolist() for n in (12, 30, 349, 7, 20)]
    g = torch.Generator().manual_seed(6)
    cond = (torch.randn(1, cfg.ar_dim, generator=g), torch.randn(1, 2 * cfg.diff_dim, generator=g))
    kw = dict(conditioning_latents=cond, use_deterministic_seed=3, max_mel_tokens=40, num_autoregressive_samples=6,
              diffusion_iterations=4)
    E = ar_engine.AREngine
    saved = E.MODE
    os.environ["TTB_AR_STEP_TEAM"] = "1"
    try:
        E.MODE = "mixed"
        got = tts.tts_batch(["x"] * 5, preset="ultra_fast", text_tokens_list=toks, **kw)
        assert set(tts.last_timings) >= {"ar_ms", "clvp_ms", "diffusion_ms", "vocoder_ms", "device_total_ms"}
        for u in range(5):
            want = tts.tts_with_preset("x", preset="ultra_fast", text_tokens=toks[u], **kw)
            assert got[u].shape == want.shape
            d = (got[u] - want).abs().max().item()
            report("tts_batch vs tts waveform u=%d" % u, d)
            assert d == 0.0
    finally:
        E.MODE = saved
        os.environ.pop("TTB_AR_STEP_TEAM", None)
    a = tts.tts_batch(["x"] * 2, preset="ultra_fast", text_tokens_list=[toks[0], toks[1]], **kw)
    graph = tts.autoregressive._dec["graph"]
    assert graph is not None
    b = tts.tts_batch(["x"] * 2, preset="ultra_fast", text_tokens_list=[toks[0], toks[1]], **kw)
    assert tts.autoregressive._dec["graph"] is graph, "the second call captured a new graph"
    for x, y in zip(a, b):
        assert x.shape[:2] == (1, 1) and torch.isfinite(x).all()
        assert torch.equal(x, y)
