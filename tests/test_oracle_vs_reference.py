"""Pins oracle/*.py against the UNMODIFIED reference modules (the copy build() places under oracle/_ref; without
it these tests skip and the committed tests/golden/* fixtures carry the pin instead)."""
import os

import numpy as np
import pytest
import torch

from tortoise_tts_b200.config import ModelConfig
from tortoise_tts_b200.synth import synth_all

pytestmark = pytest.mark.reference


@pytest.fixture(scope="module")
def small():
    from oracle.ref_build import build_reference_models
    cfg = ModelConfig.small()
    sds = synth_all(cfg, seed=0, suppress_stop=False)
    with torch.no_grad():
        models = build_reference_models(cfg, sds, kv_cache=True)
    return cfg, sds, models


TEXT = [42, 2, 194, 91, 24, 2, 243, 190, 2, 182, 37, 2, 0]  # once zero-padded, as api.py:391 does


def test_ar_teacher_forced_logits_recompute_path(small):
    """oracle teacher_forced_logits(train_consistent) == GPT2InferenceModel full-recompute forward."""
    from oracle import ar
    cfg, sds, m = small
    sd = sds["autoregressive"]
    uv = m["autoregressive"]
    torch.manual_seed(1)
    cond = torch.randn(1, cfg.ar_dim)
    codes = torch.randint(0, 8192, (2, 7))
    with torch.no_grad():
        want = ar.teacher_forced_logits(sd, cfg, cond, TEXT, codes, pos_mode="train_consistent")
        # reference: recompute path of the inference model (kv_cache off => whole sequence every call)
        inf = uv.inference_model
        inf.kv_cache = False
        text = torch.tensor(TEXT[:-1] + [0]).unsqueeze(0)  # tokens + api pad
        ti = torch.nn.functional.pad(text, (0, 1), value=0)
        ti = torch.nn.functional.pad(ti, (1, 0), value=cfg.start_text_token)
        emb = uv.text_embedding(ti) + uv.text_pos_embedding(ti)
        emb = torch.cat([cond.unsqueeze(1), emb], dim=1)
        inf.store_mel_emb(emb)
        fake = torch.full((2, emb.shape[1] + 1), 1, dtype=torch.long)
        fake[:, -1] = cfg.start_mel_token
        ids = torch.cat([fake, codes], dim=1)
        out = inf(input_ids=ids, attention_mask=torch.ones_like(ids), return_dict=True)
        got = out.logits[:, emb.shape[1]:]
        inf.kv_cache = True
    assert got.shape == want.shape
    assert (got - want).abs().max().item() < 2e-4


def test_ar_generate_matches_reference_kv_path(small):
    """With identical forced samples, oracle KV decode (ref_kv_quirk) logits == reference cached logits."""
    from oracle import ar
    cfg, sds, m = small
    sd = sds["autoregressive"]
    uv = m["autoregressive"]
    inf = uv.inference_model
    torch.manual_seed(2)
    cond = torch.randn(1, cfg.ar_dim)
    codes = torch.randint(0, 8192, (1, 5))
    with torch.no_grad():
        want = ar.teacher_forced_logits(sd, cfg, cond, TEXT, codes, pos_mode="ref_kv_quirk")
        text = torch.tensor(TEXT).unsqueeze(0)
        ti = torch.nn.functional.pad(text, (0, 1), value=0)
        ti = torch.nn.functional.pad(ti, (1, 0), value=cfg.start_text_token)
        emb = uv.text_embedding(ti) + uv.text_pos_embedding(ti)
        emb = torch.cat([cond.unsqueeze(1), emb], dim=1)
        inf.store_mel_emb(emb)
        fake = torch.full((1, emb.shape[1] + 1), 1, dtype=torch.long)
        fake[:, -1] = cfg.start_mel_token
        ids = fake
        past = None
        got = []
        for j in range(codes.shape[1] + 1):
            am = torch.ones_like(ids)
            if past is None:
                out = inf(input_ids=ids, attention_mask=am, use_cache=True, return_dict=True)
            else:
                out = inf(input_ids=ids[:, -1:], past_key_values=past, attention_mask=am, use_cache=True,
                          return_dict=True)
            past = out.past_key_values
            got.append(out.logits[:, -1])
            if j < codes.shape[1]:
                ids = torch.cat([ids, codes[:, j:j + 1]], dim=1)
        got = torch.stack(got, dim=1)
    assert (got - want).abs().max().item() < 2e-4


def test_stream_latents_match_reference_kv_path(small):
    """oracle.stream_latents == what `sample_stream` yields next to every token (stream_generator.py:982):
    `final_norm(outputs.hidden_states[-1][:, -1])` of the cached forward, fed the same forced tokens. (The generator
    itself is a transformers-4.31 `GenerationMixin` copy that does not run on the installed 5.x; the forward it calls and
    the expression it yields are exercised here directly.)"""
    from oracle import ar
    cfg, sds, m = small
    sd = sds["autoregressive"]
    uv = m["autoregressive"]
    inf = uv.inference_model
    torch.manual_seed(21)
    cond = torch.randn(1, cfg.ar_dim)
    codes = torch.randint(0, 8192, (1, 6))
    codes[0, -1] = cfg.stop_mel_token               # the stop token is yielded too
    with torch.no_grad():
        want = ar.stream_latents(sd, cfg, cond, TEXT, codes[0], pos_mode="ref_kv_quirk")
        text = torch.tensor(TEXT).unsqueeze(0)
        ids = uv.compute_embeddings(cond, text)      # stores the prompt embeddings, returns the fake input ids
        past = None
        got = []
        for j in range(codes.shape[1]):
            am = torch.ones_like(ids)
            kw = dict(attention_mask=am, use_cache=True, return_dict=True, output_hidden_states=True)
            out = inf(input_ids=ids, **kw) if past is None else inf(input_ids=ids[:, -1:], past_key_values=past, **kw)
            past = out.past_key_values
            got.append(inf.final_norm(out.hidden_states[-1][:, -1])[0])
            ids = torch.cat([ids, codes[:, j:j + 1]], dim=1)
        got = torch.stack(got, dim=0)
    assert got.shape == want.shape == (6, cfg.ar_dim)
    assert (got - want).abs().max().item() < 2e-4
    # without the KV cache the reference recomputes the sequence with positions 0..n (autoregressive.py:136-146):
    # the stream latents are then the rows of the teacher-forced latent pass
    with torch.no_grad():
        a = ar.stream_latents(sd, cfg, cond, TEXT, codes[0], pos_mode="train_consistent")
        b = ar.latents(sd, cfg, cond, TEXT, codes)[0]
    assert (a - b).abs().max().item() < 1e-5


def test_handle_chunks_matches_reference():
    """tortoise_tts_b200.api_fast.TextToSpeech.handle_chunks == api_fast.py:277-303 over a whole stream (growing decoder
    outputs, the short last chunk and the repeated flush at the end included)."""
    # the module itself pulls in wav2vec alignment etc.; the method is taken from the reference SOURCE at run time
    import ast
    from oracle.ref_shims import REFERENCE_ROOT
    src = open(os.path.join(REFERENCE_ROOT, "tortoise", "api_fast.py")).read()
    fn = [n for n in ast.walk(ast.parse(src)) if isinstance(n, ast.FunctionDef) and n.name == "handle_chunks"][0]
    ns = {"torch": torch}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), "api_fast.handle_chunks", "exec"), ns)
    ref = ns["handle_chunks"]
    from tortoise_tts_b200.api_fast import TextToSpeech as Mine
    torch.manual_seed(5)
    base = torch.randn(9000)
    for lens, ov in (((3000, 5200, 5200, 5300), 1024), ((2500, 2600, 9000), 512), ((4000,), 1024)):
        st_r = (None, None)
        st_m = (None, None)
        for n in lens:
            w = base[:n] * 0.9 + 0.01 * n / 9000.0          # a new tensor per flush, like a decoder output
            cr, pr, orr = ref(None, w.clone(), st_r[0], st_r[1], ov)
            cm, pm, om = Mine.handle_chunks(None, w.clone(), st_m[0], st_m[1], ov)
            assert torch.equal(cr, cm)
            assert (orr is None) == (om is None) and (orr is None or torch.equal(orr, om))
            st_r, st_m = (pr, orr), (pm, om)


def test_sampler_matches_hf_processors(small):
    """oracle.sample_step kept set / probabilities == HF processor chain (RepetitionPenalty ->
    Temperature -> TopK -> TopP) of the installed transformers (form identical to 4.31)."""
    from transformers.generation.logits_process import (RepetitionPenaltyLogitsProcessor, TemperatureLogitsWarper,
                                                        TopKLogitsWarper, TopPLogitsWarper)
    from oracle import ar
    torch.manual_seed(3)
    for trial in range(5):
        logits = torch.randn(1, 8194) * 3
        prev = torch.cat([torch.tensor([[1] * 10 + [8192]]), torch.randint(0, 8192, (1, 20))], dim=1)
        s = RepetitionPenaltyLogitsProcessor(2.0)(prev, logits.clone())
        s = TemperatureLogitsWarper(0.8)(prev, s)
        s = TopKLogitsWarper(50)(prev, s)
        s = TopPLogitsWarper(0.8)(prev, s)
        p = torch.softmax(s, dim=-1)[0]
        tok, kept, kp = ar.sample_step(logits[0], prev[0].tolist(), 0.5)
        ref_kept = (p > 0).nonzero().flatten()
        assert sorted(kept.tolist()) == sorted(ref_kept.tolist())
        assert (p[kept] - kp).abs().max().item() < 1e-6
        assert tok in kept.tolist()


def test_fix_autoregressive_output(small):
    from oracle import ar
    from tortoise.api import fix_autoregressive_output
    for row in ([5, 6, 7, 8193, 8193, 8193, 8193, 8193], [1, 2, 3, 4, 5, 6], [8193, 1, 2, 3], [1, 2, 3, 4, 5, 8193]):
        c = torch.tensor(row)
        want = fix_autoregressive_output(c.clone(), 8193, complain=False)
        got = ar.fix_autoregressive_output(c, 8193)
        assert torch.equal(want, got)


def test_ar_latents(small):
    from oracle import ar
    cfg, sds, m = small
    uv = m["autoregressive"]
    torch.manual_seed(4)
    cond = torch.randn(1, cfg.ar_dim)
    codes = torch.randint(0, 8192, (2, 12))
    text = torch.tensor(TEXT).unsqueeze(0)
    with torch.no_grad():
        want = uv(cond.repeat(2, 1), text.repeat(2, 1), torch.tensor([text.shape[-1]]), codes,
                  torch.tensor([codes.shape[-1] * uv.mel_length_compression]), return_latent=True, clip_inputs=False)
        got = ar.latents(sds["autoregressive"], cfg, cond, TEXT, codes)
    assert got.shape == want.shape == (2, 12, cfg.ar_dim)
    assert (got - want).abs().max().item() < 2e-4


def test_clvp_scores(small):
    from oracle import clvp
    cfg, sds, m = small
    torch.manual_seed(5)
    codes = torch.randint(0, 8192, (3, 20))
    text = torch.tensor(TEXT)
    with torch.no_grad():
        want = m["clvp"](text.unsqueeze(0).repeat(3, 1), codes, return_loss=False)
        got = clvp.scores(sds["clvp"], cfg, text, codes)
    assert (got - want).abs().max().item() < 1e-5


def test_cvvp_scores(small):
    """oracle/cvvp.py == CVVP.forward(mel_cond, codes, return_loss=False) accumulated over the conditioning clips as
    api.py:464-468 does (strict=True load of the synthetic cvvp.pth checks the key layout too)."""
    from oracle import cvvp
    cfg, sds, m = small
    torch.manual_seed(15)
    codes = torch.randint(0, 8192, (3, 23))
    auto_conds = torch.randn(1, 2, 80, 131) * 2 - 4           # [1, n_clips, 80, T] as get_conditioning_latents returns
    with torch.no_grad():
        acc = 0
        for cl in range(auto_conds.shape[1]):
            acc = acc + m["cvvp"](auto_conds[:, cl].repeat(3, 1, 1), codes, return_loss=False)
        want = acc / auto_conds.shape[1]
        got = cvvp.scores(sds["cvvp"], cfg, auto_conds, codes)
    assert (got - want).abs().max().item() < 1e-5


def test_hifigan(small):
    """oracle/hifigan.py == HifiganGenerator.inference(gpt_latents, g=speaker latent) of the api_fast path
    (hifigan_decoder.py:270-294); strict=True load of the synthetic hifidecoder.pth checks the key layout."""
    from oracle import hifigan as oh
    cfg, sds, m = small
    torch.manual_seed(16)
    lat = torch.randn(1, 9, cfg.ar_dim)
    spk = torch.randn(1, cfg.ar_dim)
    with torch.no_grad():
        want = m["hifigan"].inference(lat, spk)
        got = oh.inference(sds["hifigan"], lat, spk)
    assert got.shape == want.shape and got.shape[-1] == 256 * int(int(9 * 4) * 24000 / 22050)
    assert (got - want).abs().max().item() < 1e-5
    assert want.abs().max().item() > 0.05          # a meaningful waveform, not a saturated / vanishing one


def test_diffusion_forward_and_loop(small):
    from oracle import diffusion as od
    from tortoise.api import load_discrete_vocoder_diffuser, do_spectrogram_diffusion
    cfg, sds, m = small
    sd = sds["diffusion"]
    dm = m["diffusion"]
    torch.manual_seed(6)
    N = 10
    lat = torch.randn(1, N, cfg.ar_dim)
    cond = torch.randn(1, 2 * cfg.diff_dim)
    S = od.output_seq_len(N)
    with torch.no_grad():
        ce_ref = dm.timestep_independent(lat, cond, S, False)
        ce = od.timestep_independent(sd, cfg, lat, cond, S)
        assert (ce - ce_ref).abs().max().item() < 1e-4
        x = torch.randn(1, 100, S)
        t = torch.tensor([3979])
        for cf in (False, True):
            want = dm(x, t, precomputed_aligned_embeddings=ce_ref, conditioning_free=cf)
            got = od.forward(sd, cfg, x, t, code_emb=ce, conditioning_free=cf)
            assert (got - want).abs().max().item() < 1e-4
        # full sampling loop with the same torch RNG stream
        iters = 5
        diffuser = load_discrete_vocoder_diffuser(desired_diffusion_steps=iters, cond_free=True, cond_free_k=2.0)
        torch.manual_seed(7)
        want = do_spectrogram_diffusion(dm, diffuser, lat, cond, temperature=1.0, verbose=False)
        torch.manual_seed(7)
        noise0 = torch.randn(1, 100, S)
        step_noise = torch.stack([torch.randn(1, 100, S) for _ in range(iters)])
        got = od.spectrogram_diffusion(sd, cfg, lat, cond, noise0, step_noise, iters, True, 2.0)
    assert (got - want).abs().max().item() < 1e-3


def test_schedule_kats():
    """SURVEY App. A3 known-answer values, re-derived from the reference's SpacedDiffusion."""
    from oracle import diffusion as od
    from tortoise.api import load_discrete_vocoder_diffuser
    for iters in (30, 80, 200, 400):
        d = load_discrete_vocoder_diffuser(desired_diffusion_steps=iters)
        s = od.make_schedule(iters)
        assert list(s["timestep_map"]) == list(d.timestep_map)
        for name, arr in (("betas", d.betas), ("sqrt_recip_alphas_cumprod", d.sqrt_recip_alphas_cumprod),
                          ("sqrt_recipm1_alphas_cumprod", d.sqrt_recipm1_alphas_cumprod),
                          ("posterior_log_variance_clipped", d.posterior_log_variance_clipped),
                          ("posterior_mean_coef1", d.posterior_mean_coef1),
                          ("posterior_mean_coef2", d.posterior_mean_coef2)):
            assert np.array_equal(s[name], arr), name
        assert np.array_equal(s["log_betas"], np.log(d.betas))


def test_vocoder(small):
    from oracle import vocoder as ov
    cfg, sds, m = small
    torch.manual_seed(8)
    mel = torch.randn(1, 100, 12) * 2 - 5
    z = torch.randn(1, 64, 22)
    with torch.no_grad():
        want = m["vocoder"].inference(mel, z)
        got = ov.inference(sds["vocoder"], mel, z)
    assert got.shape == want.shape == (1, 1, 256 * 12)
    assert (got - want).abs().max().item() < 1e-4
