"""CPU: api_fast.TextToSpeech.tts_batch / tts_long and the one-row-per-sentence packing behind them — the planner at up to
256 prompt groups, tts_batch against one tts() call per text and tts_long against the concatenation, with the kernel
library replaced by the row-by-row torch emulation (tests/lib_emu.py + tests/lib_emu_grouped.py), and the argument
checks."""
import pytest
import torch

import lib_emu_grouped
from tortoise_tts_b200 import lib
from tortoise_tts_b200.ar_engine import plan_batches
from tortoise_tts_b200.config import ModelConfig
from tortoise_tts_b200.synth import synth_all


# ------------------------------------------------------------------ planner
def test_plan_one_row_per_sentence_up_to_256_groups():
    assert lib.AR_STEP_MAX_GROUPS == lib.AR_STEP_MAX_B == 256
    assert plan_batches([(1, 60)] * 40) == [list(range(40))]
    assert plan_batches([(1, 60)] * 300) == [list(range(256)), list(range(256, 300))]
    # a prompt of 353+ positions is decoded alone, in order, between the batches around it
    utts = [(1, 50)] * 100 + [(1, 353)] + [(1, 352)] * 200 + [(1, 400)]
    assert plan_batches(utts) == [list(range(100)), [100], list(range(101, 301)), [301]]


# ------------------------------------------------------------------ facade on the emulation
@pytest.fixture(scope="module")
def env():
    saved = lib_emu_grouped.install()
    cfg = ModelConfig.small()
    yield cfg, synth_all(cfg, seed=0, suppress_stop=False)
    lib_emu_grouped.uninstall(saved)


def _fast_facade(cfg, sds, monkeypatch):
    """api_fast.TextToSpeech on the CPU emulation (the constructor insists on a CUDA device: fields set by hand), with a
    fixed random voice and a short generation limit."""
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
    voice = torch.randn(1, cfg.ar_dim, generator=torch.Generator().manual_seed(7))
    monkeypatch.setattr(t, "get_random_conditioning_latents", lambda: voice)
    monkeypatch.setattr(type(cfg), "max_mel_tokens", property(lambda self: 9), raising=False)
    return t


TEXTS = [[42, 2, 194, 91, 24, 2], [7, 77, 8, 9, 100, 12, 13, 14, 15, 3, 2], [5, 6], [9, 9, 30]]
KW = dict(use_deterministic_seed=11, verbose=False)


def test_tts_batch_equals_one_tts_per_text(env, monkeypatch):
    cfg, sds = env
    t = _fast_facade(cfg, sds, monkeypatch)
    long_text = torch.randint(1, 255, (349,), generator=torch.Generator().manual_seed(2)).tolist()   # P = 354
    texts = TEXTS[:2] + [long_text] + TEXTS[2:]
    grouped, alone = [], []
    ar = t.autoregressive
    gen_grouped, gen = ar.generate_grouped, ar.generate
    monkeypatch.setattr(ar, "generate_grouped", lambda *a, **kw: grouped.append(a[2]) or gen_grouped(*a, **kw))
    monkeypatch.setattr(ar, "generate", lambda *a, **kw: alone.append(a[2]) or gen(*a, **kw))
    got = t.tts_batch(["x"] * len(texts), text_tokens_list=texts, temperature=0.7, **KW)
    assert grouped == [[1, 1], [1, 1]] and alone == [1], "two grouped batches around the long prompt decoded alone"
    assert len(got) == len(texts)
    tokens = t.last_timings["tokens"]
    assert len(tokens) == len(texts)
    for u, toks in enumerate(texts):
        want = t.tts("x", text_tokens=toks, temperature=0.7, **KW)
        assert t.last_timings["tokens"] == tokens[u]
        assert got[u].shape == want.shape and got[u].shape[:2] == (1, 1) and got[u].dtype == torch.float32
        assert torch.equal(got[u], want)


def test_tts_long_splits_and_concatenates(env, monkeypatch):
    cfg, sds = env
    t = _fast_facade(cfg, sds, monkeypatch)
    got = t.tts_long("one|two|three", text_tokens_list=TEXTS[:3], **KW)
    parts = [t.tts("x", text_tokens=toks, **KW) for toks in TEXTS[:3]]
    want = torch.cat([p.reshape(1, -1) for p in parts], dim=-1)
    assert got.device.type == "cpu" and got.shape == want.shape and got.shape[0] == 1
    assert torch.equal(got, want)
    # without '|' the text is split by split_and_recombine_text, every chunk rendered in one tts_batch call
    from tortoise_tts_b200.text import split_and_recombine_text
    text = ("This is the first sentence of a long read, and it goes on for a while so that the splitter has something "
            "to do. " * 6)
    chunks = split_and_recombine_text(text)
    assert len(chunks) > 1
    seen = []
    monkeypatch.setattr(t, "tts_batch", lambda texts, **kw: seen.append((texts, kw)) or
                        [torch.full((1, 1, 3), float(i)) for i in range(len(texts))])
    out = t.tts_long(text, use_deterministic_seed=4)
    assert len(seen) == 1 and seen[0][0] == chunks and seen[0][1]["use_deterministic_seed"] == 4
    assert torch.equal(out, torch.arange(len(chunks), dtype=torch.float32).repeat_interleave(3).reshape(1, -1))


def test_fast_batch_argument_errors(env, monkeypatch):
    cfg, sds = env
    t = _fast_facade(cfg, sds, monkeypatch)
    with pytest.raises(ValueError):
        t.tts_batch([])
    with pytest.raises(ValueError):
        t.tts_batch(["a", "b"], text_tokens_list=[[1, 2]])
    with pytest.raises(TypeError):
        t.tts_batch(["a"], text_tokens_list=[[1, 2]], no_repeat_ngram_size=2, **KW)
    with pytest.raises(TypeError):
        t.tts_batch(["a"], text_tokens=[1, 2], **KW)           # one id list per text: text_tokens_list
    with pytest.raises(ValueError):
        t.tts_batch(["a"], text_tokens_list=[[1, 2]], typical_sampling=True, typical_mass=0.0, **KW)
    with pytest.raises(ValueError):
        t.tts_long("a|b", text_tokens_list=[[1, 2]])
