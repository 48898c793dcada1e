"""GPU: the wav2vec2 aligner kernels against fp32 torch, the aligner engine against HF Wav2Vec2ForCTC, and prompt
redaction through TextToSpeech.tts."""
import math

import pytest
import torch
import torch.nn.functional as F

from gpu_util import report

pytestmark = pytest.mark.gpu
TEXT = [42, 2, 194, 91, 24, 2, 243, 190, 2, 182, 37, 2]


def _bf(t):
    return t.to(torch.bfloat16).float()


def test_wav2vec_conv0_matches_torch():
    from tortoise_tts_b200 import lib
    g = torch.Generator().manual_seed(0)
    n, C = 2 * 16000 + 7, 512
    x = (torch.randn(n, generator=g) * 0.2 + 0.05).cuda()
    w, b = torch.randn(C, 10, generator=g).cuda() * 0.3, torch.randn(C, generator=g).cuda() * 0.1
    gm, bt = 1 + torch.randn(C, generator=g).cuda() * 0.1, torch.randn(C, generator=g).cuda() * 0.1
    L0 = (n - 10) // 5 + 1
    out = torch.zeros(L0 + 1, C, dtype=torch.bfloat16, device="cuda")
    stats = torch.empty(2, device="cuda")
    lib.wav2vec_conv0(x, n, w, b, gm, bt, C, stats, out, C)
    xd = x.double()
    mean, sd = xd.mean(), torch.sqrt(xd.var() + 1e-7)
    assert abs(stats[0].item() - mean.item()) < 1e-6 and abs(stats[1].item() / sd.item() - 1) < 1e-5
    xn = ((xd - mean) / sd).float()
    y = F.conv1d(xn.reshape(1, 1, -1), w.reshape(C, 1, 10), b, stride=5)[0].t()
    want = F.gelu(F.layer_norm(y, (C,), gm, bt, 1e-5))
    err = (out[:L0].float() - want).abs().max().item()
    report("wav2vec conv0 (bf16 out)", err)
    assert err < 0.02 + 0.008 * want.abs().max().item()
    assert out[L0].abs().max().item() == 0          # rows past the output are not touched


@pytest.mark.parametrize("D", [256, 512, 1024])
@pytest.mark.parametrize("gelu", [False, True])
def test_layernorm_act(D, gelu):
    from tortoise_tts_b200 import lib
    g = torch.Generator().manual_seed(D)
    M = 37
    x = (torch.randn(M, D, generator=g) * 3 + 1).cuda()
    gm, bt = (1 + 0.1 * torch.randn(D, generator=g)).cuda(), (0.1 * torch.randn(D, generator=g)).cuda()
    of = torch.empty(M, D, device="cuda")
    ob = torch.empty(M, D, dtype=torch.bfloat16, device="cuda")
    lib.layernorm_act(x, M, D, gm, bt, gelu=gelu, out_bf16=ob, out_f32=of)
    want = F.layer_norm(x, (D,), gm, bt, 1e-5)
    if gelu:
        want = F.gelu(want)
    assert (of - want).abs().max().item() < 1e-4
    assert (ob.float() - want).abs().max().item() < 0.02 * want.abs().max().item()


def test_argmax_rows_ties_and_nan():
    from tortoise_tts_b200 import lib
    g = torch.Generator().manual_seed(1)
    for V in (37, 5001):
        x = torch.randn(64, V, generator=g)
        for r in range(0, 64, 3):                   # ties of the maximum at two or three places
            i, j = sorted(torch.randperm(V, generator=g)[:2].tolist())
            x[r, i] = x[r, j] = x[r].max() + 1
            if r % 2:
                x[r, V - 1] = x[r, i]
        x[5] = 0.25                                   # an all-equal row
        x[7, V // 2] = float("nan")                   # NaN wins, as in torch.argmax
        x[8, 3] = x[8, V - 2] = float("nan")
        xc = x.cuda()
        out = torch.empty(64, dtype=torch.int32, device="cuda")
        lib.argmax_rows(xc, 64, V, out)
        assert torch.equal(out.cpu().long(), x.argmax(-1)), V


@pytest.mark.parametrize("force_ref", [False, True])
def test_gemm_gelu_erf_epilogue(force_ref):
    from tortoise_tts_b200 import lib
    g = torch.Generator().manual_seed(2)
    M, N, K = 200, 192, 128
    A = torch.randn(M, K, generator=g).to(torch.bfloat16).cuda()
    W = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(torch.bfloat16).cuda()
    b = torch.randn(N, generator=g).cuda()
    r = torch.randn(M, N, generator=g).cuda()
    out = torch.empty(M, N, device="cuda")
    outb = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    lib.gemm(A, W, M=M, N=N, K=K, bias=b, residual=r, out_f32=out, out_bf16=outb, act=lib.ACT_GELU_ERF,
             force_ref=force_ref)
    want = F.gelu(A.float() @ W.float().t() + b) + r
    err = (out - want).abs().max().item()
    report("gemm GELU_ERF epilogue%s" % (" (SIMT)" if force_ref else ""), err)
    assert err < 1e-3
    assert (outb.float() - want).abs().max().item() < 0.05


@pytest.mark.parametrize("k,L", [(3, 101), (3, 100), (2, 77)])
def test_strided_conv_pair_view(k, L):
    """Conv1d(C, C, k, stride 2) as ttb_gemm over rows read in pairs, with an odd input length where it matters."""
    from tortoise_tts_b200 import lib
    g = torch.Generator().manual_seed(k * 1000 + L)
    C = 256
    x = _bf(torch.randn(L, C, generator=g))
    w = torch.randn(C, C, k, generator=g) / math.sqrt(C * k)
    b = torch.randn(C, generator=g) * 0.1
    buf = torch.zeros(L + 1, C, dtype=torch.bfloat16, device="cuda")
    buf[:L] = x.to(torch.bfloat16).cuda()
    taps = (k + 1) // 2
    wk = torch.zeros(C, 2 * taps, C)
    wk[:, :k] = w.permute(0, 2, 1)
    Wp = wk.reshape(C, taps * 2 * C).to(torch.bfloat16).cuda()
    Lout = (L - k) // 2 + 1
    out = torch.empty(Lout, C, device="cuda")
    lib.gemm(buf, Wp, M=Lout, N=C, K=2 * C, rows=(L + 1) // 2, taps=taps, bias=b.cuda(), out_f32=out)
    want = F.conv1d(x.t().unsqueeze(0), _bf(w), b, stride=2)[0].t()
    assert out.shape == want.shape
    err = (out.cpu() - want).abs().max().item()
    report("pair-view conv k=%d L=%d" % (k, L), err)
    assert err < 2e-3


# ---------------------------------------------------------------- engine against HF Wav2Vec2ForCTC (fp32, same GPU)
def _speechlike(n, seed):
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(n) / 24000.0
    env = 0.5 + 0.5 * torch.sin(2 * math.pi * 3.1 * t)
    x = sum(torch.sin(2 * math.pi * f * t + p) for f, p in ((180, 0.3), (410, 1.1), (1250, 2.0))) * env * 0.1
    return (x + 0.02 * torch.randn(n, generator=g)).float()


@pytest.mark.parametrize("size,seconds", [("small", 3.0), ("full", 20.0)])
def test_engine_logits_match_hf(size, seconds):
    import torchaudio
    from transformers import Wav2Vec2Config, Wav2Vec2ForCTC
    from tortoise_tts_b200.synth import synth_wav2vec
    from tortoise_tts_b200.wav2vec_engine import Wav2VecEngine
    cfg, sd, _ = synth_wav2vec(size, seed=4)
    eng = Wav2VecEngine(cfg, sd, "cuda")
    wav = _speechlike(int(seconds * 24000) + 13, 5).cuda()
    got = eng.logits(wav)
    ids = eng.ids(wav)
    m = Wav2Vec2ForCTC(Wav2Vec2Config(**cfg)).eval()
    m.load_state_dict(sd)
    m = m.cuda()
    with torch.no_grad():
        a = torchaudio.functional.resample(wav.reshape(1, -1), 24000, 16000)
        want = m((a - a.mean()) / torch.sqrt(a.var() + 1e-7)).logits[0]
    del m
    assert got.shape == want.shape
    scale = want.abs().max().item()
    err = (got - want).abs().max().item() / scale
    report("wav2vec %s %.0f s logits (of scale)" % (size, seconds), err)
    assert err < 0.03
    top2 = want.topk(2, dim=-1).values
    sure = (top2[:, 0] - top2[:, 1]) > 0.03 * scale
    assert torch.equal(ids.long()[sure], want.argmax(-1)[sure])
    report("wav2vec %s frames with a clear argmax" % size, sure.float().mean().item())


# ---------------------------------------------------------------- through the public interface
@pytest.fixture(scope="module")
def tts_small():
    from tortoise_tts_b200.api import TextToSpeech
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_all, synth_wav2vec
    cfg = ModelConfig.small()
    sds = synth_all(cfg, seed=0, suppress_stop=False)
    w_cfg, w_sd, w_vocab = synth_wav2vec("small", seed=1)
    # the random head must not emit <s> / </s> / <unk>: their multi-character spellings in the decoded string would
    # make the alignment fail (as it does in the reference), and this test is about the cut
    w_sd["lm_head.bias"][[w_vocab[t] for t in ("<s>", "</s>", "<unk>")]] = -1e4
    sds["wav2vec"] = (w_cfg, w_sd, w_vocab)
    tts = TextToSpeech(state_dicts=sds, config=cfg, kv_cache=True)
    cl = (torch.randn(1, cfg.ar_dim, generator=torch.Generator().manual_seed(2)),
          torch.randn(1, 2 * cfg.diff_dim, generator=torch.Generator().manual_seed(3)) * 0.3)
    kw = dict(text_tokens=TEXT, conditioning_latents=cl, use_deterministic_seed=5, max_mel_tokens=24,
              num_autoregressive_samples=8, diffusion_iterations=4, verbose=False, cond_free=False)
    return tts, sds, kw


def test_tts_redacts_bracketed_prompt(tts_small):
    from tortoise_tts_b200 import redaction
    tts, sds, kw = tts_small
    text = "[I am sad,] hello there, how are you"
    tts.enable_redaction = False
    full = tts.tts(text, **kw)
    assert "redaction_ms" not in tts.last_timings
    tts.enable_redaction = True
    got = tts.tts(text, **kw)
    assert "redaction_ms" in tts.last_timings and tts.aligner is not None
    report("redaction ms (small aligner, %d samples)" % full.shape[-1], tts.last_timings["redaction_ms"])
    assert got.dim() == 3 and got.shape[:2] == (1, 1)
    ids = tts.aligner.engine.ids(full.reshape(-1).cuda()).cpu().tolist()
    want = redaction.redact(full.reshape(1, -1), text, ids, redaction.CTCCharTokenizer(sds["wav2vec"][2]))
    assert torch.equal(got.reshape(1, -1), want)
    assert got.shape[-1] < full.shape[-1]
    outs = tts.tts(text, k=2, **kw)
    assert isinstance(outs, list) and len(outs) == 2 and all(o.dim() == 3 for o in outs)


def test_tts_without_redaction_is_unchanged(tts_small):
    tts, sds, kw = tts_small
    tts.enable_redaction = False
    base = tts.tts("unused", **kw)
    off = tts.tts("[I am sad,] hello", **kw)
    tts.enable_redaction = True
    plain = tts.tts("hello there", **kw)
    assert "redaction_ms" not in tts.last_timings
    assert torch.equal(base, off) and torch.equal(base, plain)


def test_missing_aligner_weights_raise(tmp_path, monkeypatch, tts_small):
    tts, sds, kw = tts_small
    monkeypatch.setenv("HF_HOME", str(tmp_path))
    monkeypatch.delenv("HF_HUB_CACHE", raising=False)
    monkeypatch.delenv("TORTOISE_WAV2VEC_DIR", raising=False)
    monkeypatch.delenv("TORTOISE_WAV2VEC_VOCAB", raising=False)
    saved, aligner = tts._wav2vec, tts.aligner
    tts._wav2vec, tts.aligner = None, None
    try:
        with pytest.raises(FileNotFoundError, match="enable_redaction=False"):
            tts.tts("[x] y", **kw)
    finally:
        tts._wav2vec, tts.aligner = saved, aligner
