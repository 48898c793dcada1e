"""CPU: the streaming batch of the api_fast path — the flush rule shared by tts_stream and tts_stream_batch on fake token
streams, AREngine.generate_grouped_stream with latent capture, HifiganEngine.inference_batch, tts_stream_batch /
tts_long_stream against tts_stream, tts_batch with one voice per text, and the argument checks, with the kernel library
replaced by the row-by-row torch emulation (tests/lib_emu.py + lib_emu_grouped.py + lib_emu_stream.py)."""
import pytest
import torch

import lib_emu_stream
from test_fast_batch_host import _fast_facade
from tortoise_tts_b200 import api_fast
from tortoise_tts_b200.api_fast import stream_flushes
from tortoise_tts_b200.config import ModelConfig
from tortoise_tts_b200.synth import synth_all


# ------------------------------------------------------------------ the flush rule
def _token_stream(stop_at, cap, first, block):
    """The (n, ended) yields of AREngine.generate_stream for a row that samples its stop token as token number `stop_at`
    (1-based; None = never) and is capped at `cap` tokens."""
    out, have, target = [], 1, max(1, first)
    while True:
        have = max(have, min(target, cap))
        if stop_at is not None and stop_at <= have:
            return out + [(stop_at, True)]
        if have >= cap:
            return out + [(have, True)]
        out.append((have, False))
        target = have + max(1, block)


def _schedule(chunk, cap):
    return (max(chunk, 60), chunk) if chunk > 0 else (cap, cap)


CASES = [  # (stop_at, cap, stream_chunk_size, [(tokens covered, is_end) of every flush])
    (30, 440, 40, [(30, True)]),                                        # stops before the first buffer is full
    (75, 440, 40, [(60, False), (75, True)]),                           # stops inside a block
    (None, 130, 40, [(60, False), (100, False), (130, True)]),          # reaches its cap
    (None, 140, 40, [(60, False), (100, False), (140, False), (140, True)]),   # due and ended: two flushes
    (140, 440, 40, [(60, False), (100, False), (140, False), (140, True)]),
    (None, 200, 0, [(200, True)]),                                      # stream_chunk_size <= 0: one flush at the end
    (57, 440, -3, [(57, True)]),
    (None, 300, 70, [(70, False), (140, False), (210, False), (280, False), (300, True)]),   # first flush at 70, not 60
]


@pytest.mark.parametrize("stop_at,cap,chunk,want", CASES)
def test_flush_rule_gives_the_reference_sequence(stop_at, cap, chunk, want):
    flushes, flushed = [], 0
    for n, ended in _token_stream(stop_at, cap, *_schedule(chunk, cap)):
        for is_end in stream_flushes(n, flushed, ended, chunk):
            flushes.append((n, is_end))
            flushed = n
    assert flushes == want


@pytest.mark.parametrize("stop_at,cap,chunk,want", CASES)
def test_tts_stream_flushes_by_the_rule(stop_at, cap, chunk, want, monkeypatch):
    """tts_stream driven by a fake token stream flushes exactly where the rule says (its output did not change when the
    rule moved into stream_flushes)."""
    t = api_fast.TextToSpeech.__new__(api_fast.TextToSpeech)
    t.device, t.kv_cache = torch.device("cpu"), True
    toks = [1, 2, 3]
    P = len(toks) + 1 + 4
    monkeypatch.setattr(api_fast, "STREAM_MAX_LENGTH", P + cap)
    seen = {}

    class FakeAR:
        def generate_stream(self, auto, toks, n_max, first, block, **kw):
            assert n_max == cap and (first, block) == _schedule(chunk, cap)
            for n, ended in _token_stream(stop_at, cap, first, block):
                yield torch.arange(n, dtype=torch.int32), ended

        def stream_latents(self, auto, toks, codes):
            return torch.full((codes.numel(), 1), float(codes.numel()))

    class FakeHifi:
        def inference(self, lat, auto):
            seen.setdefault("n", []).append(int(lat.shape[0]))
            return torch.ones(4096 * lat.shape[0])

    t.autoregressive, t.hifi_decoder = FakeAR(), FakeHifi()
    monkeypatch.setattr(t, "_auto_latent", lambda v: torch.zeros(4))
    chunks = list(t.tts_stream("x", text_tokens=toks, stream_chunk_size=chunk, use_deterministic_seed=1, verbose=False))
    assert seen["n"] == [n for n, _ in want] and len(chunks) == len(want)


# ------------------------------------------------------------------ engines and facade on the emulation
@pytest.fixture(scope="module")
def env():
    saved = lib_emu_stream.install()
    cfg = ModelConfig.small()
    yield cfg, synth_all(cfg, seed=0, suppress_stop=False)
    lib_emu_stream.uninstall(saved)


TEXTS = [[42, 2, 194, 91, 24, 2], [7, 77, 8, 9, 100, 12, 13, 14, 15, 3, 2], [5, 6], [9, 9, 30]]
KW = dict(use_deterministic_seed=11, verbose=False, stream_chunk_size=6)


def _short_streams(monkeypatch):
    """Streams of 24-33 tokens with a first flush at 10 tokens, so that the emulation runs in seconds."""
    monkeypatch.setattr(api_fast, "STREAM_MAX_LENGTH", 40)
    monkeypatch.setattr(api_fast, "FIRST_BUFFER", 10)


def _rel(a, b):
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-6)


def test_grouped_stream_captures_the_stream_latents(env):
    """Per row: the tokens generate_stream samples alone, and captured latents that match stream_latents over them."""
    from tortoise_tts_b200.ar_engine import AREngine
    cfg, sds = env
    eng = AREngine(sds["autoregressive"], cfg, device="cpu")
    g = torch.Generator().manual_seed(3)
    voices = [torch.randn(cfg.ar_dim, generator=g) for _ in TEXTS]
    toks = [t + [0] for t in TEXTS]
    caps = [14, 9, 17, 12]
    us = [torch.rand(1, c, generator=g) for c in caps]
    yields = list(eng.generate_grouped_stream(voices, toks, caps, 5, 4, uniforms_list=us, use_graph=False))
    codes, ended, lat = yields[-1]
    assert all(ended) and [y[0][0].numel() for y in yields] == [5, 9, 13, 14]
    assert lat.shape == (len(TEXTS), max(caps), cfg.ar_dim)
    for u in range(len(TEXTS)):
        alone = [c for c, _ in eng.generate_stream(voices[u], toks[u], caps[u], 5, 4, uniforms=us[u], use_graph=False)]
        assert torch.equal(codes[u], alone[-1])
        n = codes[u].numel()
        want = eng.stream_latents(voices[u], toks[u], codes[u])
        assert _rel(lat[u, :n], want) < 2e-3


def test_inference_batch_equals_one_inference_per_row(env):
    from tortoise_tts_b200.hifigan_engine import HifiganEngine
    cfg, sds = env
    hifi = HifiganEngine(sds["hifigan"], cfg, device="cpu")
    g = torch.Generator().manual_seed(1)
    lat = torch.randn(3, 7, cfg.ar_dim, generator=g)
    spk = torch.randn(3, cfg.ar_dim, generator=g)
    got = hifi.inference_batch(lat, spk)
    assert got.shape == (3, 256 * hifi.output_frames(7))
    # the emulation's batched matmuls sum in another order than one item's (1.9e-5 here); on the GPU every item runs the
    # kernel one item runs, and tests/test_gpu_stream_batch.py pins bit identity
    for r in range(3):
        want = hifi.inference(lat[r], spk[r])
        assert (got[r] - want).abs().max().item() < 1e-4
    hifi.BATCH_FRAMES = 1                  # one item per pass
    assert (hifi.inference_batch(lat, spk) - got).abs().max().item() < 1e-4


def _stream_rows(out, R):
    rows = [[] for _ in range(R)]
    for u, chunk, last in out:
        assert not rows[u] or not rows[u][-1][1], "a chunk after the last one of stream %d" % u
        rows[u].append((chunk, last))
    return rows


def test_stream_batch_matches_tts_stream_per_text(env, monkeypatch):
    cfg, sds = env
    t = _fast_facade(cfg, sds, monkeypatch)
    _short_streams(monkeypatch)
    out = list(t.tts_stream_batch(["x"] * len(TEXTS), text_tokens_list=TEXTS, temperature=0.7, **KW))
    tim = t.last_timings
    rows = _stream_rows(out, len(TEXTS))
    assert len(tim["tokens"]) == len(TEXTS)
    for u, toks in enumerate(TEXTS):
        want = list(t.tts_stream("x", text_tokens=toks, temperature=0.7, **KW))
        got = rows[u]
        assert [len(c) for c, _ in got] == [len(c) for c in want]
        assert [last for _, last in got] == [False] * (len(want) - 1) + [True]
        assert len(want) >= 4
        # only the latent source differs: captured in the decode steps vs one teacher-forced pass per flush
        for (c, _), w in zip(got, want):
            assert (c - w).abs().max().item() < 2e-2


def test_long_stream_is_the_concatenation_in_order(env, monkeypatch):
    cfg, sds = env
    t = _fast_facade(cfg, sds, monkeypatch)
    _short_streams(monkeypatch)
    got = list(t.tts_long_stream("one|two|three", text_tokens_list=TEXTS[:3], **KW))
    want = [c for toks in TEXTS[:3] for c in t.tts_stream("x", text_tokens=toks, **KW)]
    assert [len(c) for c in got] == [len(c) for c in want]
    assert all(c.dim() == 1 for c in got)
    assert max((a - b).abs().max().item() for a, b in zip(got, want)) < 2e-2


def test_long_stream_batches_and_streams_long_prompts_alone(env, monkeypatch):
    """More sentences than one batch takes, and a prompt too long for the batch: consecutive batches, tts_stream for
    that sentence, every chunk in playback order, one seed for all."""
    cfg, sds = env
    t = _fast_facade(cfg, sds, monkeypatch)
    from tortoise_tts_b200 import lib
    monkeypatch.setattr(lib, "AR_STEP_MAX_GROUPS", 2)
    calls = []

    def fake_batch(texts, text_tokens_list=None, use_deterministic_seed=None, **kw):
        calls.append(("batch", [tt[0] for tt in text_tokens_list], use_deterministic_seed))
        R = len(texts)
        # interleaved and out of order: row R-1 first
        for i in range(2):
            for u in reversed(range(R)):
                yield u, torch.tensor([float(text_tokens_list[u][0]), float(i)]), i == 1

    def fake_stream(text, text_tokens=None, use_deterministic_seed=None, **kw):
        calls.append(("alone", [text_tokens[0]], use_deterministic_seed))
        yield torch.tensor([float(text_tokens[0]), 0.0])
        yield torch.tensor([float(text_tokens[0]), 1.0])

    monkeypatch.setattr(t, "tts_stream_batch", fake_batch)
    monkeypatch.setattr(t, "tts_stream", fake_stream)
    toks = [[1], [2], [3] + [7] * 400, [4], [5], [6]]
    got = list(t.tts_long_stream("a|b|c|d|e|f", text_tokens_list=toks, use_deterministic_seed=9, verbose=False))
    assert [c.tolist() for c in got] == [[float(s), float(i)] for s in range(1, 7) for i in range(2)]
    assert calls == [("batch", [1, 2], 9), ("alone", [3], 9), ("batch", [4, 5], 9), ("batch", [6], 9)]


def test_tts_batch_with_one_voice_per_text(env, monkeypatch):
    """conditioning_latents_list: entry u equals tts(texts[u], voice_samples=clips_u) when latent u is what
    get_conditioning_latents(clips_u) returns."""
    cfg, sds = env
    t = _fast_facade(cfg, sds, monkeypatch)
    g = torch.Generator().manual_seed(2)
    voices = {"a": torch.randn(1, cfg.ar_dim, generator=g), "b": torch.randn(1, cfg.ar_dim, generator=g)}
    monkeypatch.setattr(t, "get_conditioning_latents", lambda clips, return_mels=False: voices[clips])
    which = ["a", "b", "b", "a"]
    got = t.tts_batch(["x"] * len(TEXTS), text_tokens_list=TEXTS, conditioning_latents_list=[voices[w] for w in which],
                      use_deterministic_seed=11, verbose=False)
    for u, toks in enumerate(TEXTS):
        want = t.tts("x", voice_samples=which[u], text_tokens=toks, use_deterministic_seed=11, verbose=False)
        assert torch.equal(got[u], want)


def test_stream_batch_argument_errors(env, monkeypatch):
    cfg, sds = env
    t = _fast_facade(cfg, sds, monkeypatch)
    lat = torch.zeros(1, cfg.ar_dim)
    with pytest.raises(ValueError):
        t.tts_stream_batch([])
    with pytest.raises(ValueError):
        t.tts_stream_batch(["a", "b"], text_tokens_list=[[1, 2]])
    with pytest.raises(ValueError):
        t.tts_stream_batch(["a", "b"], text_tokens_list=[[1], [2]], conditioning_latents_list=[lat])
    with pytest.raises(ValueError):
        t.tts_stream_batch(["a"], voice_samples=["clip"], text_tokens_list=[[1]], conditioning_latents_list=[lat])
    with pytest.raises(ValueError):
        t.tts_stream_batch(["a"] * 257, text_tokens_list=[[1]] * 257)
    with pytest.raises(ValueError):                                      # P = 349 + 1 + 4 = 354 > 352
        t.tts_stream_batch(["a", "b"], text_tokens_list=[[1], [5] * 349])
    t.tts_stream_batch(["a"], text_tokens_list=[[5] * 347])             # P = 352 is accepted
    with pytest.raises(TypeError):
        t.tts_stream_batch(["a"], text_tokens_list=[[1]], no_repeat_ngram_size=2)
    with pytest.raises(TypeError):
        t.tts_stream_batch(["a"], text_tokens_list=[[1]], typical_sampling=True)
    with pytest.raises(TypeError):
        t.tts_stream_batch(["a"], text_tokens_list=[[1]], text_tokens=[1])      # one id list per text
    with pytest.raises(ValueError):
        t.tts_batch(["a"], voice_samples=["clip"], text_tokens_list=[[1]], conditioning_latents_list=[lat])
    with pytest.raises(ValueError):
        t.tts_batch(["a", "b"], text_tokens_list=[[1], [2]], conditioning_latents_list=[lat])
    with pytest.raises(ValueError):
        t.tts_long_stream("a|b", text_tokens_list=[[1]])
