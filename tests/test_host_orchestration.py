"""CPU: the stage engines' HOST orchestration (weight packing, op order, strides) checked against the golden vectors
with the kernel library replaced by a torch emulation (tests/lib_emu.py). The kernels themselves are checked on the
GPU by tests/test_gpu_*.py; this catches host-side mistakes without a GPU."""
import os

import pytest
import torch

import lib_emu
from tortoise_tts_b200.config import ModelConfig
from tortoise_tts_b200.synth import synth_all

GOLD = os.path.join(os.path.dirname(__file__), "golden", "small_v1.pt")


@pytest.fixture(scope="module")
def env():
    saved = lib_emu.install()
    cfg = ModelConfig.small()
    yield cfg, synth_all(cfg, seed=0, suppress_stop=False), torch.load(GOLD)
    lib_emu.uninstall(saved)


def _rel(a, b):
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-6)


def test_ar_engine(env):
    from tortoise_tts_b200.ar_engine import AREngine
    from oracle import ar
    cfg, sds, g = env
    eng = AREngine(sds["autoregressive"], cfg, device="cpu")
    text = g["text"].tolist()
    for mode, key in (("ref_kv_quirk", "ar_logits_kv"), ("train_consistent", "ar_logits_recompute")):
        got = eng.teacher_forced_logits(g["ar_cond"], text, g["ar_codes"], pos_mode=mode)
        assert _rel(got, g[key]) < 0.03
    assert _rel(eng.latents(g["ar_cond"], text, g["lat_codes"]), g["latents"]) < 0.03
    # decode loop: logits seen by the sampler must equal teacher-forced logits of the produced sequence
    torch.manual_seed(0)
    u = torch.rand(3, 6)
    codes = eng.generate(g["ar_cond"], text, 3, 6, uniforms=u, use_graph=False).long()
    with torch.no_grad():
        lg = ar.teacher_forced_logits(sds["autoregressive"], cfg, g["ar_cond"], text, codes[:, :-1], "ref_kv_quirk")
    agree = 0
    for b in range(3):
        seen = {1, cfg.start_mel_token}
        for n in range(6):
            tok, kept, _ = ar.sample_step(lg[b, n], seen, float(u[b, n]))
            assert int(codes[b, n]) in kept.tolist()
            agree += int(tok == int(codes[b, n]))
            seen.add(int(codes[b, n]))
    assert agree >= 13


def test_ar_stream(env):
    """Block-wise decoding of ONE sequence (the token stream of the api_fast path) == the batch decode loop, block
    boundaries / end-of-stream handling, and the stream latents against the oracle (pinned against the reference's cached
    forward in tests/test_oracle_vs_reference.py)."""
    from tortoise_tts_b200.ar_engine import AREngine
    from oracle import ar
    cfg, sds, g = env
    eng = AREngine(sds["autoregressive"], cfg, device="cpu")
    text = g["text"].tolist()
    torch.manual_seed(1)
    u = torch.rand(1, 20)
    full = eng.generate(g["ar_cond"], text, 1, 20, uniforms=u, use_graph=False)[0]
    hit = (full == cfg.stop_mel_token).nonzero()
    n_end = int(hit[0]) + 1 if hit.numel() else 20
    out = list(eng.generate_stream(g["ar_cond"], text, 20, 6, 4, uniforms=u, use_graph=False))
    want_bounds = [b for b in (6, 10, 14, 18) if b < n_end] + [n_end]
    assert [int(c.numel()) for c, _ in out] == want_bounds
    assert [e for _, e in out] == [False] * (len(out) - 1) + [True]
    for c, _ in out:
        assert torch.equal(c, full[: c.numel()])
    codes = out[-1][0].long()
    for mode in ("ref_kv_quirk",):
        got = eng.stream_latents(g["ar_cond"], text, codes)
        with torch.no_grad():
            want = ar.stream_latents(sds["autoregressive"], cfg, g["ar_cond"], text, codes, pos_mode=mode)
        assert got.shape == want.shape == (codes.numel(), cfg.ar_dim)
        assert _rel(got, want) < 0.03


def test_ar_two_chains_equal_one(env, monkeypatch):
    """TTB_AR_CHAINS=2 (two half-batches decoded as independent chains inside one step) must reproduce the one-chain
    result bit for bit: the sampler is keyed by the candidate's own row of the uniforms table and its own KV cache."""
    from tortoise_tts_b200.ar_engine import AREngine
    cfg, sds, g = env
    text = g["text"].tolist()
    torch.manual_seed(2)
    u = torch.rand(4, 7)
    monkeypatch.setattr(AREngine, "MODE", "mixed")
    monkeypatch.setattr(AREngine, "CHAINS_MIN_B", 2)
    outs = []
    for n in (1, 2):
        monkeypatch.setattr(AREngine, "CHAINS", n)
        eng = AREngine(sds["autoregressive"], cfg, device="cpu")
        tr = []
        codes = eng.generate(g["ar_cond"], text, 4, 7, uniforms=u, use_graph=False, trace_logits=tr)
        assert len(eng._dec["chains"]) == n and eng._dec["mode"] == "mixed"
        outs.append((codes, torch.stack(tr, 1)))
    assert torch.equal(outs[0][0], outs[1][0])
    # (the emulation's torch matmuls round differently for 2 and 4 rows; the kernels are row-independent)
    assert (outs[0][1] - outs[1][1]).abs().max().item() < 1e-3


def _fast_facade(cfg, sds):
    """api_fast.TextToSpeech on the CPU emulation (the constructor insists on a CUDA device: fields set by hand)."""
    from tortoise_tts_b200 import api_fast
    from tortoise_tts_b200.ar_engine import AREngine
    from tortoise_tts_b200.hifigan_engine import HifiganEngine
    t = api_fast.TextToSpeech.__new__(api_fast.TextToSpeech)
    t.cfg, t.device, t.kv_cache, t._sds = cfg, torch.device("cpu"), True, sds
    t.autoregressive = AREngine(sds["autoregressive"], cfg, device="cpu")
    t.hifi_decoder = HifiganEngine(sds["hifigan"], cfg, device="cpu")
    t.rlg_auto = t._conditioning = t._tokenizer = None
    t.models_dir = None
    t.last_timings = {}
    return t


def test_api_fast_tts_and_stream(env, monkeypatch):
    """Host logic of the api_fast facade (SURVEY 8f row 3) on the emulated kernels: `tts` = one sequence -> latents of
    the raw codes -> HiFiGAN; `tts_stream` = the reference's buffering rule (first max(chunk, first_buffer) tokens, then
    every chunk, once more at the end), every flush decoding ALL latents so far, `handle_chunks` cutting and
    cross-fading. Checked against a literal restatement of api_fast.py:396-420 driven by the oracle."""
    from tortoise_tts_b200 import api_fast
    from oracle import ar, hifigan as oh
    cfg, sds, g = env
    t = _fast_facade(cfg, sds)
    text = g["text"].tolist()[:-1]              # the facade pads once itself
    toks = text + [0]
    P = len(toks) + 4
    monkeypatch.setattr(api_fast, "STREAM_MAX_LENGTH", P + 30)
    monkeypatch.setattr(api_fast, "FIRST_BUFFER", 12)
    voice = torch.randn(1, cfg.ar_dim)
    monkeypatch.setattr(t, "get_random_conditioning_latents", lambda: voice)
    chunks = list(t.tts_stream("unused", text_tokens=text, use_deterministic_seed=3, stream_chunk_size=8,
                               overlap_wav_len=256, verbose=False))
    # the same tokens, from the engine (sampling parity is test_ar_engine's business)
    gen = torch.Generator(device="cpu")
    gen.manual_seed(3)
    u = torch.rand(1, 30, generator=gen)
    codes = t.autoregressive.generate(voice.reshape(-1), toks, 1, 30, uniforms=u, use_graph=False)[0].long()
    hit = (codes == cfg.stop_mel_token).nonzero()
    n = int(hit[0]) + 1 if hit.numel() else 30
    want, buf, first, prev, tail = [], 0, 12, None, None
    with torch.no_grad():
        for i in list(range(n)) + [None]:        # None = StopIteration of the token generator
            if i is not None:
                buf += 1
            if i is None or buf >= max(8, first):
                first = 0
                m = n if i is None else i + 1
                lat = ar.stream_latents(sds["autoregressive"], cfg, voice, toks, codes[:m], "ref_kv_quirk")
                wav = oh.inference(sds["hifigan"], lat.unsqueeze(0), voice)[0, 0]
                c, prev, tail = t.handle_chunks(wav, prev, tail, 256)
                buf = 0
                want.append(c)
    assert len(chunks) == len(want) and len(want) >= 3
    for a, b in zip(chunks, want):
        assert a.shape == b.shape
        assert (a - b).abs().max().item() < 0.05, (a - b).abs().max().item()   # bf16 GEMM operands in the GPT trunk
    # the pieces join into (almost) the whole utterance: everything but a cross-fade tail that is never handed out
    assert sum(c.numel() for c in chunks) >= want[-1].numel()
    # ---- tts(): raw codes incl. the stop token -> UnifiedVoice latents -> decoder
    monkeypatch.setattr(type(cfg), "max_mel_tokens", property(lambda self: 25), raising=False)
    try:
        wav = t.tts("unused", text_tokens=text, use_deterministic_seed=3, verbose=False)
    finally:
        monkeypatch.undo()
    nt = t.last_timings["tokens"]
    gen.manual_seed(3)
    u = torch.rand(1, 24, generator=gen)
    codes = t.autoregressive.generate(voice.reshape(-1), toks, 1, 24, uniforms=u, use_graph=False).long()
    assert nt == (int((codes[0] == cfg.stop_mel_token).nonzero()[0]) + 1 if (codes[0] == cfg.stop_mel_token).any() else 24)
    with torch.no_grad():
        lat = ar.latents(sds["autoregressive"], cfg, voice, toks, codes[:, :nt])
        ref = oh.inference(sds["hifigan"], lat, voice)
    assert wav.shape == ref.shape
    assert (wav - ref).abs().max().item() < 0.05


def test_clvp_engine(env):
    from tortoise_tts_b200.clvp_engine import CLVPEngine
    cfg, sds, g = env
    got = CLVPEngine(sds["clvp"], cfg, device="cpu").scores(g["text"].tolist(), g["clvp_codes"])
    assert (got - g["clvp_scores"]).abs().max().item() < 0.03


def test_diffusion_engine(env):
    from tortoise_tts_b200.diffusion_engine import DiffusionEngine
    cfg, sds, g = env
    eng = DiffusionEngine(sds["diffusion"], cfg, device="cpu")
    S = g["code_emb"].shape[-1]
    ce = eng.timestep_independent(g["diff_latents"][0], g["diff_cond"][0], S)
    assert _rel(ce.t(), g["code_emb"][0]) < 0.03
    got_c, got_u = eng.forward_once(g["diff_x"][0], 3979, ce)
    assert _rel(got_c, g["diff_fwd_cond"][0]) < 0.03 and _rel(got_u, g["diff_fwd_uncond"][0]) < 0.03
    mel = eng.sample(g["diff_latents"][0], g["diff_cond"][0], g["diff_iters"], g["diff_noise0"][0],
                     g["diff_step_noise"][:, 0], cond_free=True, cond_free_k=2.0, use_graph=False)
    # bf16 operand rounding alone (this emulation IS the fp32 oracle with bf16-rounded GEMM operands) moves the final
    # mel by ~1.0 of its 13.8 range through the 153x eps->x0 gain of the first DDPM steps: that is the noise floor
    # the GPU tolerance in tests/test_gpu_stages.py is derived from.
    err = (mel - g["diff_mel"][0]).abs().max().item()
    rms = (mel - g["diff_mel"][0]).pow(2).mean().sqrt().item()
    assert err < 1.5 and rms < 0.3, (err, rms)


def test_diffusion_engine_fused_groupnorm_statistics(env, monkeypatch):
    """Full-width denoiser (C = 1024: 32 channels per group, the case where the GEMM epilogue leaves the GroupNorm
    statistics for the GroupNorm that follows): one cond + uncond evaluation against the oracle with the fused statistics
    and with the separate statistics pass that shapes outside the fused condition take. The emulated groupnorm_apply
    uses ONLY the partials the emulated gemm stored, so a block that consumes stale partials fails here."""
    from tortoise_tts_b200.diffusion_engine import DiffusionEngine
    from tortoise_tts_b200.synth import synth_diffusion
    from oracle import diffusion as od
    cfg = ModelConfig.medium()
    sd = synth_diffusion(cfg, 0)
    torch.manual_seed(7)
    N, S = 10, 43                                      # S % 32 != 0: ragged last row block
    lat = torch.randn(N, cfg.ar_dim)
    cond = torch.randn(2 * cfg.diff_dim) * 0.3
    x = torch.randn(1, 100, S)
    with torch.no_grad():
        ce = od.timestep_independent(sd, cfg, lat.unsqueeze(0), cond.unsqueeze(0), S)
        want_c = od.forward(sd, cfg, x, torch.tensor([1000]), code_emb=ce)
        want_u = od.forward(sd, cfg, x, torch.tensor([1000]), conditioning_free=True)
    outs = {}
    for fused in (1, 0):
        if not fused:
            monkeypatch.setattr(DiffusionEngine, "_gnp", lambda self, S, ws: {})
        eng = DiffusionEngine(sd, cfg, device="cpu")
        ce_g = eng.timestep_independent(lat, cond, S)
        assert _rel(ce_g.t(), ce[0]) < 0.03
        got_c, got_u = eng.forward_once(x[0], 1000, ce_g)
        assert _rel(got_c, want_c[0]) < 0.03 and _rel(got_u, want_u[0]) < 0.03, fused
        outs[fused] = (got_c, got_u)
    # (fp32 statistics summed in a different order flip a few bf16 roundings of the normalised operand: ~0.3 %)
    assert _rel(outs[1][0], outs[0][0]) < 0.01 and _rel(outs[1][1], outs[0][1]) < 0.01


def test_cvvp_engine(env):
    """CVVP re-ranker (SURVEY 8f row 4): strided conv front-end, both CollapsingTransformers, pooling commuted with the
    last 1x1 conv, clip average folded into one latent -- against oracle/cvvp.py, kernels emulated."""
    from tortoise_tts_b200.cvvp_engine import CVVPEngine
    from oracle import cvvp as oc
    cfg, sds, g = env
    torch.manual_seed(9)
    codes = torch.randint(0, 8192, (5, 37))
    auto_conds = torch.randn(1, 2, 80, 151) * 2 - 4
    eng = CVVPEngine(sds["cvvp"], cfg, device="cpu")
    with torch.no_grad():
        want = oc.scores(sds["cvvp"], cfg, auto_conds, codes)
        want_c = oc.cond_latent(sds["cvvp"], cfg, auto_conds[:, 1])
    got_c = eng.cond_latent(auto_conds[0, 1])
    assert (got_c - want_c).abs().max().item() < 0.03
    got = eng.scores(auto_conds, codes, chunk=2)
    assert (got - want).abs().max().item() < 0.03, (got, want)
    with pytest.raises(IndexError):
        eng.scores(auto_conds, torch.full((1, 4), 8192))


def test_hifigan_engine(env):
    """HiFiGAN decoder of the api_fast path (SURVEY 8f row 3): interpolation lengths, weight-norm folding, the
    ConvTranspose -> 3-tap GEMM rewrite, dilated taps, split operands, ResBlock streams -- against oracle/hifigan.py."""
    from tortoise_tts_b200.hifigan_engine import HifiganEngine
    from oracle import hifigan as oh
    cfg, sds, g = env
    torch.manual_seed(12)
    lat = torch.randn(11, cfg.ar_dim)
    spk = torch.randn(cfg.ar_dim)
    eng = HifiganEngine(sds["hifigan"], cfg, device="cpu")
    with torch.no_grad():
        want = oh.inference(sds["hifigan"], lat.unsqueeze(0), spk.unsqueeze(0))[0, 0]
    got = eng.inference(lat, spk)
    assert got.shape == want.shape == (256 * eng.output_frames(11),)
    assert (got - want).abs().max().item() < 2e-3, (got - want).abs().max().item()


def test_vocoder_engine(env):
    from tortoise_tts_b200.vocoder_engine import VocoderEngine
    cfg, sds, g = env
    wav = VocoderEngine(sds["vocoder"], cfg, device="cpu").inference(g["voc_mel"][0], g["voc_z"][0])
    err = (wav - g["voc_wav"][0, 0]).abs().max().item()
    assert err < 0.03, err


def test_conditioning_engine(env):
    """Conditioning front-end (tables, resampling bank, STFT framing, strided convs, clip / position means) against the
    oracle, kernels emulated: catches host-side mistakes in table construction and layouts."""
    from tortoise_tts_b200.conditioning_engine import ConditioningEngine, RandomLatentEngine
    from tortoise_tts_b200.synth import synth_rlg
    from oracle import conditioning as oc
    cfg, sds, g = env
    torch.manual_seed(4)
    clips = [(torch.randn(1, n) * 0.2).clamp(-1, 1) for n in (140000, 60000)]
    mel_norms = -(torch.rand(80) * 5 + 1)
    eng = ConditioningEngine(sds["autoregressive"], sds["diffusion"], cfg, device="cpu", mel_norms=mel_norms)
    starts = [23, None]
    with torch.no_grad():
        want_ar = oc.ar_conditioning_latent(sds["autoregressive"], cfg, clips, mel_norms, starts)
        want_df = oc.diffusion_conditioning_latent(sds["diffusion"], cfg, clips)
    got_ar, mels = eng.ar_latent(clips, starts, return_mels=True)
    w0 = oc.format_conditioning_clip(clips[0], 23)
    assert (mels[0, 0] - oc.torch_mel_spectrogram(w0, mel_norms)[0]).abs().max() < 2e-3
    assert _rel(got_ar, want_ar) < 0.03
    got_df, dmels = eng.diffusion_latent(clips, return_mels=True)
    s0 = oc.resample_22k_24k(clips[0])[..., :oc.DIFF_COND_LENGTH]
    assert (dmels[0, 0] - oc.tacotron_mel(s0)[0]).abs().max() < 2e-3
    assert _rel(got_df, want_df) < 0.03
    sd = synth_rlg(64, 0)
    r = torch.randn(1, 64)
    assert (RandomLatentEngine(sd, 64, "cpu")(r) - oc.random_latent(sd, r)).abs().max() < 1e-5
