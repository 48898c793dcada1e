"""GPU: every stage at the PRODUCTION shapes of BASELINE configs[2] (T = 169 text tokens, N = 430 mel tokens, S = 1872 mel
frames, full depth: 30-layer GPT-2, 20-layer CLVP encoders, 10+3+3-layer denoiser) against the oracle (oracle/*.py, fp32).

The oracle is plain torch; here it runs ON THE GPU in true fp32 (TF32 off, tests/conftest.py) under
`torch.device("cuda")` so that the full-size comparison takes seconds instead of the ~25 s per unit of the CPU baseline.
Nothing else about it changes: same functions, same state dicts.

Tolerances (relative to the scale of each quantity, bf16 GEMM operands / fp32 everything else): logits, scores, eps
prediction as in tests/test_gpu_stages.py (3 % bound, ~0.6 % measured at small sizes). The 200-step sampled mel gets its
own stated bound, see test_sampled_mel_200_steps.
"""
import json
import os

import pytest
import torch

from gpu_util import check_sampled_mel, report

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rel(a, b):
    return (a.float() - b.float()).abs().max().item() / max(b.float().abs().max().item(), 1e-6)


def _rel_live(got, want):
    """Logit error relative to the scale of the LIVE logits: the synthetic checkpoint pins the start / stop token biases at
    -1e4 (SURVEY 8d), which would otherwise set the scale and hide a 1e4 x larger error."""
    live = want.float() > -1e3
    g, w = got.float()[live], want.float()[live]
    return (g - w).abs().max().item() / max(w.abs().max().item(), 1e-6)


def _cuda_sd(sd):
    return {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in sd.items()}


def _tokens():
    with open(os.path.join(ROOT, "tests", "golden", "bench_text_tokens.json")) as f:
        return json.load(f)["para53"]["tokens"]


@pytest.fixture(scope="module")
def full():
    from tortoise_tts_b200.config import ModelConfig
    return ModelConfig.full()


def test_ar_teacher_forced_full_depth_T169_N430(full):
    """Rows a1/a2: logits at all 430 decode positions of 2 candidates behind the 174-position prompt, 30 layers."""
    from tortoise_tts_b200.synth import synth_autoregressive
    from tortoise_tts_b200.ar_engine import AREngine
    from oracle import ar
    cfg = full
    sd = synth_autoregressive(cfg, 0, True)
    toks = _tokens() + [0]
    torch.manual_seed(0)
    cond = torch.randn(1, cfg.ar_dim) * 0.5
    codes = torch.randint(0, 8192, (2, 430))
    got = AREngine(sd, cfg).teacher_forced_logits(cond, toks, codes)
    sdc = _cuda_sd(sd)
    with torch.no_grad(), torch.device("cuda"):
        want = ar.teacher_forced_logits(sdc, cfg, cond.cuda(), toks, codes.cuda())
    r = _rel_live(got, want.to(got.device))
    report("prod AR teacher-forced logits T=169 N=430 L=30 (live-logit scale)", r)
    assert r < 0.03


def test_ar_decode_loop_full_depth_prompt174(full):
    """The KV-cached decode loop itself (prefill P = 174, then the one-kernel step) at full depth: logits the sampler sees
    at 48 consecutive steps vs the oracle's teacher-forced logits of the produced sequence."""
    from tortoise_tts_b200.synth import synth_autoregressive
    from tortoise_tts_b200.ar_engine import AREngine
    from oracle import ar
    cfg = full
    sd = synth_autoregressive(cfg, 0, True)
    toks = _tokens() + [0]
    torch.manual_seed(1)
    cond = torch.randn(1, cfg.ar_dim) * 0.5
    B, N = 4, 48
    u = torch.rand(B, N)
    tr = []
    codes = AREngine(sd, cfg).generate(cond, toks, B, N, uniforms=u, trace_logits=tr).long()
    seen = torch.stack(tr, 1)
    sdc = _cuda_sd(sd)
    with torch.no_grad(), torch.device("cuda"):
        want = ar.teacher_forced_logits(sdc, cfg, cond.cuda(), toks, codes[:, :-1].cuda())
    r = _rel_live(seen, want.to(seen.device))
    report("prod AR decode-loop logits P=174 L=30 (48 steps, live-logit scale)", r)
    assert r < 0.03


def test_clvp_full_depth_L430(full):
    """Row a5: scores of 2 candidates of 430 codes, 20-layer encoders."""
    from tortoise_tts_b200.synth import synth_clvp
    from tortoise_tts_b200.clvp_engine import CLVPEngine
    from oracle import clvp
    cfg = full
    sd = synth_clvp(cfg, 0)
    toks = _tokens() + [0]
    torch.manual_seed(2)
    codes = torch.randint(0, 8192, (2, 430))
    got = CLVPEngine(sd, cfg).scores(toks, codes)
    sdc = _cuda_sd(sd)
    with torch.no_grad(), torch.device("cuda"):
        want = clvp.scores(sdc, cfg, torch.tensor(toks), codes.cuda())
    e = (got - want).abs().max().item()
    report("prod CLVP scores L=430 depth=20 abs", e)
    assert e < 0.03


def test_denoiser_forward_full_depth_S1872(full):
    """Rows a9/a10: timestep_independent from 430 latents and one cond + one uncond denoiser evaluation at S = 1872."""
    from tortoise_tts_b200.synth import synth_diffusion
    from tortoise_tts_b200.diffusion_engine import DiffusionEngine
    from oracle import diffusion as od
    cfg = full
    sd = synth_diffusion(cfg, 0)
    torch.manual_seed(3)
    N = 430
    S = N * 4 * 24000 // 22050
    lat = torch.randn(N, cfg.ar_dim)
    cond = torch.randn(2 * cfg.diff_dim) * 0.3
    x = torch.randn(1, 100, S)
    eng = DiffusionEngine(sd, cfg)
    ce_g = eng.timestep_independent(lat, cond, S)
    sdc = _cuda_sd(sd)
    with torch.no_grad(), torch.device("cuda"):
        ce = od.timestep_independent(sdc, cfg, lat.cuda().unsqueeze(0), cond.cuda().unsqueeze(0), S)
        r = _rel(ce_g.t(), ce[0])
        report("prod diffusion code_emb N=430 S=1872", r)
        assert r < 0.03
        for t in (3979, 1000):
            got_c, got_u = eng.forward_once(x[0], t, ce_g)
            tt = torch.tensor([t])
            want_c = od.forward(sdc, cfg, x.cuda(), tt, code_emb=ce)
            want_u = od.forward(sdc, cfg, x.cuda(), tt, conditioning_free=True)
            rc, ru = _rel(got_c, want_c[0]), _rel(got_u, want_u[0])
            report("prod diffusion forward S=1872 t=%d cond" % t, rc)
            report("prod diffusion forward S=1872 t=%d uncond" % t, ru)
            assert rc < 0.03 and ru < 0.03


def test_sampled_mel_200_steps(full):
    """Row a11: the 200-step CFG sampling loop at full depth against the oracle's p_sample_loop with the SAME injected
    noise, step by step (S = 374 = the 10-word utterance, so that 400 fp32 oracle forwards stay in tens of seconds).

    What is bounded and why. One eps evaluation differs by ~0.6 % (bf16 operands). The update x0 = clamp(sqrt(1/abar) x -
    sqrt(1/abar - 1) eps) multiplies that by up to 153 at t = 3999 before the clamp (utils/diffusion.py:420-425), and the
    learned-range variance feeds the difference back through the noise term; with random weights the two trajectories
    therefore separate early and then evolve as two samples of the same chain. The hard checks are per-step on the FIRST
    steps (where both still see the same x): |dx| after step 1 <= 3 % of |x|; and distributional on the final mel
    (gpu_util.check_sampled_mel: rms <= 0.3, 99.9th percentile <= 1.5 of the 13.8 mel range = 1.5 x the drift measured
    when the fp32 oracle itself is run with bf16-rounded GEMM operands, tests/test_host_orchestration.py; max <= 4.0). The full per-step max / rms series goes to the
    parity log (gpu_util.report)."""
    from tortoise_tts_b200.synth import synth_diffusion
    from tortoise_tts_b200.diffusion_engine import DiffusionEngine
    from oracle import diffusion as od
    cfg = full
    sd = synth_diffusion(cfg, 0)
    torch.manual_seed(4)
    N, iters = 86, 200
    S = N * 4 * 24000 // 22050
    lat = torch.randn(N, cfg.ar_dim)
    cond = torch.randn(2 * cfg.diff_dim) * 0.3
    noise0 = torch.randn(100, S)
    step_noise = torch.randn(iters, 100, S)
    eng = DiffusionEngine(sd, cfg)
    mel_g, trace_g = eng.sample(lat, cond, iters, noise0, step_noise, cond_free=True, cond_free_k=2.0, return_trace=True)
    mel_graph = eng.sample(lat, cond, iters, noise0, step_noise, cond_free=True, cond_free_k=2.0, use_graph=True)
    assert (mel_graph - mel_g).abs().max().item() < 1e-3, "graph replay and eager loop disagree"
    sdc = _cuda_sd(sd)
    with torch.no_grad(), torch.device("cuda"):
        ce = od.timestep_independent(sdc, cfg, lat.cuda().unsqueeze(0), cond.cuda().unsqueeze(0), S)
        x_o, trace_o = od.p_sample_loop(sdc, cfg, ce, noise0.cuda().unsqueeze(0), step_noise.cuda().unsqueeze(1), iters,
                                        cond_free=True, cond_free_k=2.0, return_trace=True)
        mel_o = od.denormalize_tacotron_mel(x_o)[0]
    series = []
    for c in range(iters):
        d = trace_g[c] - trace_o[c][0]
        series.append((d.abs().max().item(), d.pow(2).mean().sqrt().item(), trace_o[c][0].abs().max().item()))
    for c in (0, 1, 2, 5, 10, 50, 100, 150, 199):
        report("prod 200-step sampler |dx| max at call %d" % c, series[c][0], rms=series[c][1], x_absmax=series[c][2])
    assert series[0][0] <= 0.03 * max(series[0][2], 1.0), series[0]
    check_sampled_mel("prod 200-step sampled mel", mel_g, mel_o)
    # the two chains must agree in distribution: per-channel mean of the final mel
    dm = (mel_g.mean(-1) - mel_o.mean(-1)).abs().max().item()
    report("prod 200-step sampled mel per-channel mean diff", dm)
    assert dm < 0.5


def test_vocoder_S1872():
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_vocoder
    from tortoise_tts_b200.vocoder_engine import VocoderEngine
    from oracle import vocoder as ov
    cfg = ModelConfig.full()
    sd = synth_vocoder(cfg, 0)
    torch.manual_seed(5)
    S = 1872
    mel = torch.randn(100, S) * 2 - 5
    z = torch.randn(64, S + 10)
    wav = VocoderEngine(sd, cfg).inference(mel, z)
    sdc = _cuda_sd(sd)
    with torch.no_grad(), torch.device("cuda"):
        want = ov.inference(sdc, mel.cuda().unsqueeze(0), z.cuda().unsqueeze(0))[0, 0]
    e = (wav - want).abs().max().item()
    report("prod vocoder waveform S=1872 abs", e)
    assert e < 0.03
