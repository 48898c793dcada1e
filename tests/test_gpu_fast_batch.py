"""GPU: up to 256 prompt groups in the decode step (one per row) and api_fast.TextToSpeech.tts_batch on top of them.

The attention phase with 17 to 256 prompt prefixes against fp32 torch; one-row utterances decoded as one batch against
generate() of each utterance alone (bit for bit where the step is row-independent) and against the CPU oracle at full
depth; tts_batch against one tts() call per text."""
import os

import pytest
import torch

from gpu_util import report
from test_gpu_tts_batch import _grouped_step, _rel

pytestmark = pytest.mark.gpu

PH_ATTN = 4


def _prompts(n, seed, lo=13, hi=352):
    g = torch.Generator().manual_seed(seed)
    Ps = torch.randint(lo, hi + 1, (n,), generator=g).tolist()
    Ps[0], Ps[-1] = lo, hi                     # both ends of the range in every grouping
    return Ps


def _mixed_sizes(seed):
    g = torch.Generator().manual_seed(seed)
    sizes = []
    while sum(sizes) < 230:
        sizes.append(int(torch.randint(1, 6, (1,), generator=g)))
    return sizes


GROUPINGS = {  # name: (group sizes, prompt lengths)
    "17x1": ([1] * 17, _prompts(17, 1)),
    "64x1": ([1] * 64, _prompts(64, 2)),
    "256x1": ([1] * 256, _prompts(256, 3)),
    "mixed": (_mixed_sizes(4), _prompts(len(_mixed_sizes(4)), 5)),
}


@pytest.mark.parametrize("name", list(GROUPINGS))
@pytest.mark.parametrize("nc", [1, 215])
@pytest.mark.parametrize("compact", [False, True])
def test_many_groups_attention_phase(name, nc, compact):
    """The attention phase (debug_phase_mask = 4, one layer) with one prompt prefix per row (or per few rows) against
    fp32 torch: every row attends to [its group's prefix | own KV | new token]; only the new cache slot is written."""
    sizes, Ps = GROUPINGS[name]
    H, L, Nmax, layer = 16, 2, 430, 1
    D = H * 64
    hd, t, groups = _grouped_step(sizes, Ps, H, L, Nmax, nc, seed=nc + len(sizes), attn_compact=compact)
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
    report("many-group attention %s (%d groups, %d rows) nc=%d compact=%d" % (name, len(sizes), B, nc, compact), worst)
    assert worst < 8e-3                        # the bound of test_step_attention_phase (bf16 softmax weights in P V)


def _texts(n, seed, longest=347):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(8, 120, (n,), generator=g).tolist()
    lens[n // 2] = longest                     # one prompt at the 352-position limit
    return [torch.randint(1, 255, (k,), generator=g).tolist() + [0] for k in lens]


@pytest.mark.parametrize("n_utt,chains", [(64, 1), (64, 2), (200, 1), (200, 2)])
def test_one_row_utterances_bit_identical_to_each_alone(n_utt, chains):
    """TTB_AR_STEP_TEAM=1, mixed step: n one-row utterances decoded as one batch (one prompt group per row) give every
    row the codes and logits of generate() of that utterance alone, bit for bit, eager and as a graph replay."""
    from tortoise_tts_b200 import ar_engine
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_all
    cfg = ModelConfig.medium()
    sd = synth_all(cfg, seed=1, suppress_stop=True)["autoregressive"]
    torch.manual_seed(0)
    texts, cond = _texts(n_utt, n_utt), torch.randn(1, cfg.ar_dim)
    N = 16
    us = [torch.rand(1, N) for _ in range(n_utt)]
    E = ar_engine.AREngine
    saved = (E.MODE, E.CHAINS, E.CHAINS_MIN_B)
    os.environ["TTB_AR_STEP_TEAM"] = "1"
    try:
        E.MODE, E.CHAINS, E.CHAINS_MIN_B = "mixed", chains, 64
        eng = E(sd, cfg)
        tr = []
        got = eng.generate_grouped(cond, texts, [1] * n_utt, N, uniforms_list=us, trace_logits=tr)
        assert len(eng._dec["chains"]) == chains and len(eng._dec["groups"]) == n_utt
        seen = torch.stack([x.cpu() for x in tr], 1)
        got_g = eng.generate_grouped(cond, texts, [1] * n_utt, N, uniforms_list=us, use_graph=True)
        assert all(torch.equal(a, b) for a, b in zip(got, got_g)), "graph replay of the grouped step differs from eager"
        worst = 0.0
        for u in range(n_utt):
            tr1 = []
            want = eng.generate(cond, texts[u], 1, N, uniforms=us[u], trace_logits=tr1)
            assert eng._dec["mode"] == "mixed"
            assert torch.equal(got[u].cpu(), want.cpu()), "codes of utterance %d differ" % u
            worst = max(worst, (seen[u:u + 1] - torch.stack([x.cpu() for x in tr1], 1)).abs().max().item())
        report("%d one-row utterances vs alone, max |logit difference| chains=%d" % (n_utt, chains), worst)
        assert worst == 0.0
    finally:
        E.MODE, E.CHAINS, E.CHAINS_MIN_B = saved
        os.environ.pop("TTB_AR_STEP_TEAM", None)


def test_fused_step_with_24_groups_matches_each_alone():
    """The one-kernel step with 24 one-row groups against each utterance decoded alone by the same step: within bf16
    noise of the live-logit scale on the common prefix of identical tokens; graph replay == eager."""
    from tortoise_tts_b200 import ar_engine
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_all
    cfg = ModelConfig.medium()
    sd = synth_all(cfg, seed=1, suppress_stop=True)["autoregressive"]
    torch.manual_seed(1)
    n_utt, N = 24, 12
    texts, cond = _texts(n_utt, 9), torch.randn(1, cfg.ar_dim)
    us = [torch.rand(1, N) for _ in range(n_utt)]
    E = ar_engine.AREngine
    saved = E.MODE
    try:
        E.MODE = "fused"
        eng = E(sd, cfg)
        tr = []
        got = eng.generate_grouped(cond, texts, [1] * n_utt, N, uniforms_list=us, trace_logits=tr)
        assert eng._dec["mode"] == "fused"
        seen = torch.stack([x.cpu() for x in tr], 1)
        got_g = eng.generate_grouped(cond, texts, [1] * n_utt, N, uniforms_list=us, use_graph=True)
        assert all(torch.equal(a, b) for a, b in zip(got, got_g)), "graph replay of the fused grouped step differs"
        worst = 0.0
        for u in range(n_utt):
            tr1 = []
            want = eng.generate(cond, texts[u], 1, N, uniforms=us[u], trace_logits=tr1).cpu()
            l0 = torch.stack([x.cpu() for x in tr1], 1)
            live = l0[0, 0].abs() < 1e3
            scale = l0[..., live].abs().max().item()
            same = (got[u][0].cpu() == want[0]).long().cumprod(0)
            n_cmp = min(N, int(same.sum()) + 1)
            worst = max(worst, (seen[u, :n_cmp][:, live] - l0[0, :n_cmp][:, live]).abs().max().item() / scale)
        report("fused step, 24 one-row groups vs alone (rel. to the live-logit scale)", worst)
        assert worst < 0.02
    finally:
        E.MODE = saved


def test_many_groups_full_depth_vs_oracle():
    """30 layers, full width, 20 one-row utterances with different prompts in one batch (more groups than the step took
    before): the logits every row sees against the CPU oracle teacher-forced on that row's prompt and codes (fp32),
    within 3 % of the live-logit scale."""
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_autoregressive
    from tortoise_tts_b200.ar_engine import AREngine
    from oracle import ar
    cfg = ModelConfig.full()
    sd = synth_autoregressive(cfg, 2, True)
    torch.manual_seed(0)
    n_utt, N = 20, 5
    g = torch.Generator().manual_seed(3)
    texts = [torch.randint(1, 255, (int(k),), generator=g).tolist() + [0]
             for k in torch.randint(8, 90, (n_utt,), generator=g)]
    cond = torch.randn(1, cfg.ar_dim)
    us = [torch.rand(1, N) for _ in range(n_utt)]
    eng = AREngine(sd, cfg)
    tr = []
    got = eng.generate_grouped(cond, texts, [1] * n_utt, N, uniforms_list=us, trace_logits=tr)
    assert len(eng._dec["groups"]) == n_utt
    seen = torch.stack([x.cpu() for x in tr], 1)
    worst = 0.0
    for u in range(n_utt):
        with torch.no_grad():
            want = ar.teacher_forced_logits(sd, cfg, cond, texts[u], got[u].cpu().long()[:, :-1], "ref_kv_quirk")
        live = want[0, 0].abs() < 1e3
        scale = want[..., live].abs().max().item()
        worst = max(worst, (seen[u:u + 1][..., live] - want[..., live]).abs().max().item() / scale)
    report("20-group full-depth decode logits vs oracle (rel. to the live-logit scale)", worst)
    assert worst < 0.03


def _fast_facade():
    from tortoise_tts_b200.api_fast import TextToSpeech
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_all
    cfg = ModelConfig.small()
    return TextToSpeech(state_dicts=synth_all(cfg, seed=0, suppress_stop=False), config=cfg, kv_cache=True), cfg


def test_fast_tts_batch_equals_tts_per_text():
    """TTB_AR_MODE=mixed with one warp per stream: api_fast tts_batch of 22 texts (one with a prompt of 354 positions,
    decoded alone between two grouped batches) returns exactly the waveforms of one tts() call per text. With the
    default step: finite waveforms whose lengths follow each text's token count, and a second call replays the captured
    grouped step."""
    from tortoise_tts_b200 import ar_engine
    tts, cfg = _fast_facade()
    g = torch.Generator().manual_seed(5)
    lens = torch.randint(5, 60, (22,), generator=g).tolist()
    lens[9] = 349
    toks = [torch.randint(1, 255, (n,), generator=g).tolist() for n in lens]
    kw = dict(use_deterministic_seed=3, verbose=False)
    E = ar_engine.AREngine
    saved = E.MODE
    os.environ["TTB_AR_STEP_TEAM"] = "1"
    try:
        E.MODE = "mixed"
        got = tts.tts_batch(["x"] * len(toks), text_tokens_list=toks, **kw)
        tim = tts.last_timings
        assert set(tim) >= {"ar_ms", "prefill_ms", "latents_ms", "hifigan_ms", "device_total_ms", "tokens"}
        assert 0.0 < tim["prefill_ms"] < tim["ar_ms"] < tim["device_total_ms"]
        tokens = tim["tokens"]
        worst = 0.0
        for u in range(len(toks)):
            want = tts.tts("x", text_tokens=toks[u], **kw)
            assert tts.last_timings["tokens"] == tokens[u]
            assert got[u].shape == want.shape
            worst = max(worst, (got[u] - want).abs().max().item())
        report("api_fast tts_batch vs tts waveforms (22 texts)", worst)
        assert worst == 0.0
    finally:
        E.MODE = saved
        os.environ.pop("TTB_AR_STEP_TEAM", None)
    short = [t for i, t in enumerate(toks) if i != 9]
    a = tts.tts_batch(["x"] * len(short), text_tokens_list=short, **kw)
    graph = tts.autoregressive._dec["graph"]
    assert graph is not None and len(tts.autoregressive._dec["groups"]) == len(short)
    ta = tts.last_timings["tokens"]
    b = tts.tts_batch(["x"] * len(short), text_tokens_list=short, **kw)
    assert tts.autoregressive._dec["graph"] is graph, "the second call captured a new graph"
    auto = tts.get_random_conditioning_latents().float().reshape(-1)
    for u, (x, y) in enumerate(zip(a, b)):
        assert x.shape[:2] == (1, 1) and torch.isfinite(x).all()
        assert torch.equal(x, y)
        with torch.no_grad():
            n_samples = tts.hifi_decoder.inference(torch.zeros(ta[u], cfg.ar_dim, device="cuda"), auto).numel()
        assert x.shape[-1] == n_samples
