"""GPU: the streaming batch of the api_fast path — latent capture in the decode step (ttb_ar_capture_latents) against the
teacher-forced latent passes, its effect on the codes and on the captured step graph, HifiganEngine.inference_batch
against one inference() per row, and tts_stream_batch / tts_long_stream / tts_batch with one voice per text against
the per-text calls.

Bounds (DESIGN §5): the captured latents come from the KV-cached decode steps, the reference values from one
teacher-forced trunk pass over the same tokens; both round their GEMM operands to bf16 in a different order, so they
agree to the drift of the decode-step parity tests (3 % of the latents' scale), not bit for bit. The stream waveforms
differ only through that latent source."""
import os

import pytest
import torch

from gpu_util import report
from test_gpu_conditioning import _clips

pytestmark = pytest.mark.gpu

LATENT_REL = 3e-2       # captured vs recomputed latents, max abs error / max |latent|
WAVE_ABS = 5e-2         # stream chunks, captured vs recomputed latents (waveforms in [-1, 1])


def _rel(a, b):
    return (a.float() - b.float()).abs().max().item() / max(b.float().abs().max().item(), 1e-6)


def _raise_stop_logit(tts, cfg, voice, per_step=0.004):
    """Raises the stop token's mel_head bias of the loaded engine so that the sampler (temperature 0.8, top-k 50, top-p
    0.8) draws it with probability about `per_step` per token, averaged over the teacher-forced logits of 200 random
    codes: rows then end at different lengths (the synthetic model alone never samples its stop token in a stream)."""
    ar, stop = tts.autoregressive, cfg.stop_mel_token
    g = torch.Generator().manual_seed(1)
    toks = torch.randint(1, 255, (30,), generator=g).tolist() + [0]
    codes = torch.randint(0, 8192, (1, 200), generator=g)
    with torch.no_grad():
        lg = ar.teacher_forced_logits(voice, toks, codes)[0].float().cpu()
    best = None
    for b in torch.arange(0.0, 30.01, 0.25).tolist():
        s = lg.clone()
        s[:, stop] += b
        v, i = (s / 0.8).topk(50, dim=-1)
        p = torch.softmax(v, -1)
        keep = (p.cumsum(-1) - p) < 0.8
        keep[:, 0] = True
        pk = p * keep
        ps = ((pk / pk.sum(-1, keepdim=True)) * (i == stop)).sum(-1).mean().item()
        if best is None or abs(ps - per_step) < abs(best[1] - per_step):
            best = (b, ps)
    ar.w.b_head[stop] += best[0]
    return best


def _max_abs(got, want):
    return max(((a - b).abs().max().item() for a, b in zip(got, want) if a.numel()), default=0.0)


@pytest.mark.parametrize("pos_mode", ["ref_kv_quirk", "train_consistent"])
def test_capture_matches_the_latent_passes_and_leaves_the_codes(pos_mode):
    """Full widths (D = 1024), two layers, six rows with their own voices and prompts: the captured latents against
    stream_latents (kv_cache=True) / latents (kv_cache=False) over the same codes; the codes with capture on equal the
    codes with capture off bit for bit; the captured step graph has one more launch per decode chain, and capture off
    captures the step it captured before."""
    from tortoise_tts_b200.ar_engine import AREngine
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_autoregressive
    cfg = ModelConfig.medium()
    eng = AREngine(synth_autoregressive(cfg, 0, False), cfg)
    g = torch.Generator().manual_seed(8)
    lens = [12, 40, 7, 90, 25, 61]
    toks = [torch.randint(1, 255, (n,), generator=g).tolist() + [0] for n in lens]
    voices = [torch.randn(cfg.ar_dim, generator=g).cuda() for _ in lens]
    N = 120
    us = [torch.rand(1, N, generator=g).cuda() for _ in lens]
    kw = dict(pos_mode=pos_mode, temperature=0.8, top_k=50, top_p=0.8, repetition_penalty=2.0)
    off = eng.generate_grouped(voices, toks, [1] * len(lens), N, uniforms_list=us, **kw)
    calls_off = eng._dec["graph_calls"]
    chains = len(eng._dec["chains"])
    last = None
    for last in eng.generate_grouped_stream(voices, toks, N, 40, 40, uniforms_list=us, **kw):
        pass
    codes, ended, lat = last
    calls_on = eng._dec["graph_calls"]
    assert calls_on == calls_off + chains
    again = eng.generate_grouped(voices, toks, [1] * len(lens), N, uniforms_list=us, **kw)
    assert eng._dec["graph_calls"] == calls_off
    worst = 0.0
    for u in range(len(lens)):
        n = codes[u].numel()
        assert ended[u]
        assert torch.equal(codes[u], off[u][0, :n]) and torch.equal(off[u], again[u])
        if pos_mode == "ref_kv_quirk":
            want = eng.stream_latents(voices[u], toks[u], codes[u])
        else:
            want = eng.latents(voices[u], toks[u], codes[u].reshape(1, -1))[0]
        worst = max(worst, _rel(lat[u, :n], want))
    report("captured vs recomputed latents (%s, D=1024, 2 layers)" % pos_mode, worst)
    assert worst < LATENT_REL


def test_inference_batch_bit_identical_to_inference():
    """Full-size HiFiGAN: rows of two lengths with distinct speakers, in one pass and in passes of two rows."""
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.hifigan_engine import HifiganEngine
    from tortoise_tts_b200.synth import synth_hifigan
    cfg = ModelConfig.full()
    hifi = HifiganEngine(synth_hifigan(cfg, 0), cfg)
    g = torch.Generator().manual_seed(4)
    with torch.no_grad():
        for L, R in ((60, 5), (137, 3)):
            lat = (torch.randn(R, L, cfg.ar_dim, generator=g) * 0.5).cuda()
            spk = torch.randn(R, cfg.ar_dim, generator=g).cuda()
            got = hifi.inference_batch(lat, spk)
            for r in range(R):
                want = hifi.inference(lat[r], spk[r])
                assert got[r].shape == want.shape
                assert torch.equal(got[r], want), "row %d of %d at L=%d" % (r, R, L)
            saved = hifi.BATCH_FRAMES
            hifi.BATCH_FRAMES = 2 * hifi.output_frames(L)
            try:
                assert torch.equal(hifi.inference_batch(lat, spk), got)
            finally:
                hifi.BATCH_FRAMES = saved


@pytest.fixture(scope="module")
def fast():
    from tortoise_tts_b200.api_fast import TextToSpeech
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_all
    cfg = ModelConfig.small()
    tts = TextToSpeech(state_dicts=synth_all(cfg, seed=0, suppress_stop=False), config=cfg, kv_cache=True)
    clips = [_clips(seed=4), _clips(lengths=(90000,), seed=9)]
    voices = []
    for c in clips:
        # the conditioning crops long clips at positions drawn from the seeded `random`, as tts(voice_samples=...) does
        # after seeding with use_deterministic_seed: seed the same way to get the latent tts() gets
        tts.deterministic_state(3)
        voices.append(tts.get_conditioning_latents(c))
    bias, per_step = _raise_stop_logit(tts, cfg, voices[0].float().reshape(-1))
    report("stop logit raised by %.2f: draw probability per step" % bias, per_step)
    return tts, cfg, clips, voices


def _one_warp_mixed():
    from tortoise_tts_b200 import ar_engine
    E = ar_engine.AREngine
    saved = E.MODE
    os.environ["TTB_AR_STEP_TEAM"] = "1"
    E.MODE = "mixed"

    def restore():
        E.MODE = saved
        os.environ.pop("TTB_AR_STEP_TEAM", None)
    return restore


def _recorded_codes(tts, name):
    """Wraps AREngine.<name> to keep the codes of its last yield."""
    ar = tts.autoregressive
    fn = getattr(ar, name)
    box = {}

    def wrapped(*a, **kw):
        for y in fn(*a, **kw):
            box["codes"] = y[0]
            yield y
    setattr(ar, name, wrapped)
    return box, lambda: delattr(ar, name)


def test_stream_batch_equals_tts_stream_per_text(fast):
    """TTB_AR_MODE=mixed, one warp per stream: 12 texts (three with prompts of 352 positions, capped at 148 tokens), two
    voices, with a stop logit that ends some rows early. Every row: the tokens, chunk count and chunk lengths of
    tts_stream(texts[u], voice_samples=clips of its voice); the samples within WAVE_ABS."""
    tts, cfg, clips, voices = fast
    g = torch.Generator().manual_seed(6)
    lens = torch.randint(5, 60, (12,), generator=g).tolist()
    lens[2] = lens[7] = lens[11] = 347
    toks = [torch.randint(1, 255, (n,), generator=g).tolist() for n in lens]
    which = [u % 2 for u in range(12)]
    kw = dict(use_deterministic_seed=3, verbose=False)
    restore = _one_warp_mixed()
    box, unwrap = _recorded_codes(tts, "generate_grouped_stream")
    try:
        out = list(tts.tts_stream_batch(["x"] * 12, text_tokens_list=toks,
                                        conditioning_latents_list=[voices[w] for w in which], **kw))
        tim = tts.last_timings
        batch_codes = box["codes"]
        unwrap()
        assert set(tim) >= {"ar_ms", "hifigan_ms", "device_total_ms", "tokens"}
        assert 0.0 < tim["ar_ms"] < tim["device_total_ms"] and 0.0 < tim["hifigan_ms"] < tim["device_total_ms"]
        box1, unwrap1 = _recorded_codes(tts, "generate_stream")
        worst, kinds = 0.0, set()
        for u in range(12):
            got = [(c, last) for v, c, last in out if v == u]
            want = list(tts.tts_stream("x", voice_samples=clips[which[u]], text_tokens=toks[u], **kw))
            assert torch.equal(batch_codes[u], box1["codes"]), "tokens of row %d" % u
            n, cap = batch_codes[u].numel(), 500 - (lens[u] + 5)
            assert tim["tokens"][u] == n
            kinds.add("cap" if n == cap else "stop")
            assert [len(c) for c, _ in got] == [len(c) for c in want], "chunks of row %d" % u
            assert [last for _, last in got] == [False] * (len(want) - 1) + [True]
            worst = max(worst, _max_abs([c for c, _ in got], want))
        unwrap1()
        report("tts_stream_batch vs tts_stream chunks (12 texts, %s)" % sorted(kinds), worst)
        assert kinds == {"cap", "stop"}, "the texts should include rows that stop and rows that reach their cap"
        assert worst < WAVE_ABS
    finally:
        restore()


def test_long_stream_equals_tts_stream_in_order(fast):
    tts, cfg, clips, voices = fast
    g = torch.Generator().manual_seed(2)
    toks = [torch.randint(1, 255, (n,), generator=g).tolist() for n in (30, 12, 55, 20)]
    kw = dict(use_deterministic_seed=3, verbose=False, voice_samples=clips[0], stream_chunk_size=30)
    got = list(tts.tts_long_stream("a|b|c|d", text_tokens_list=toks, **kw))
    want = [c for t in toks for c in tts.tts_stream("x", text_tokens=t, **kw)]
    assert [len(c) for c in got] == [len(c) for c in want]
    worst = _max_abs(got, want)
    report("tts_long_stream vs tts_stream chunks in order", worst)
    assert worst < WAVE_ABS


def test_tts_batch_with_two_voices_equals_tts(fast):
    tts, cfg, clips, voices = fast
    g = torch.Generator().manual_seed(9)
    toks = [torch.randint(1, 255, (n,), generator=g).tolist() for n in (20, 44, 9, 31, 57, 15)]
    which = [0, 1, 1, 0, 1, 0]
    kw = dict(use_deterministic_seed=3, verbose=False)
    restore = _one_warp_mixed()
    try:
        got = tts.tts_batch(["x"] * len(toks), text_tokens_list=toks,
                            conditioning_latents_list=[voices[w] for w in which], **kw)
        for u in range(len(toks)):
            want = tts.tts("x", voice_samples=clips[which[u]], text_tokens=toks[u], **kw)
            assert got[u].shape == want.shape and torch.equal(got[u], want), "text %d" % u
    finally:
        restore()
