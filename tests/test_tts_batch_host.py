"""CPU: tts_batch and the grouped decode behind it (AREngine.generate_grouped) — the packing planner, the prompt groups
each decode chain sees, the argument checks, and tts_batch against one tts() call per text with the kernel library
replaced by the row-by-row torch emulation (tests/lib_emu.py + tests/lib_emu_grouped.py)."""
import pytest
import torch

import lib_emu_grouped
from tortoise_tts_b200.ar_engine import plan_batches, clip_groups
from tortoise_tts_b200.config import ModelConfig
from tortoise_tts_b200.synth import synth_all


# ------------------------------------------------------------------ planner
def test_plan_packs_consecutive_utterances_in_order():
    # 16 candidates each (ultra_fast): 16 utterances fill one batch of 256 rows, the 17th opens the next
    assert plan_batches([(16, 100)] * 17) == [list(range(16)), [16]]
    # 96 candidates each (fast): two per batch, the third would pass 256 rows
    assert plan_batches([(96, 50)] * 5) == [[0, 1], [2, 3], [4]]
    # exactly 256 rows fit
    assert plan_batches([(128, 10), (128, 10), (1, 10)]) == [[0, 1], [2]]


def test_plan_caps_groups_and_rows():
    assert plan_batches([(1, 20)] * 40, max_groups=16) == [list(range(16)), list(range(16, 32)), list(range(32, 40))]
    assert plan_batches([(3, 20)] * 5, max_rows=7) == [[0, 1], [2, 3], [4]]
    for batch in plan_batches([(n, 30) for n in (100, 60, 90, 7, 200, 56, 1)]):
        assert sum((100, 60, 90, 7, 200, 56, 1)[u] for u in batch) <= 256


def test_plan_decodes_oversize_utterances_alone():
    # more than 256 candidates (tts() default 512) or a prompt longer than 352 positions: a batch of its own, in order
    assert plan_batches([(16, 100), (16, 353), (16, 100), (16, 100)]) == [[0], [1], [2, 3]]
    assert plan_batches([(16, 100), (512, 100), (16, 100)]) == [[0], [1], [2]]
    assert plan_batches([(256, 352), (256, 352)]) == [[0], [1]]
    with pytest.raises(ValueError):
        plan_batches([(0, 10)])


# ------------------------------------------------------------------ chain clipping
def test_clip_groups_rebases_to_the_chain():
    a, b, c = object(), object(), object()
    groups = [(0, 50, 13, a), (50, 100, 174, b), (100, 128, 352, c)]
    # two chains of 64 rows: the middle group straddles the split and appears in both with its own prefix
    assert clip_groups(groups, 0, 64) == [(0, 50, 13, a), (50, 64, 174, b)]
    assert clip_groups(groups, 64, 128) == [(0, 36, 174, b), (36, 64, 352, c)]
    assert clip_groups(groups, 0, 128) == groups
    assert clip_groups([(0, 64, 20, a), (64, 128, 30, b)], 64, 128) == [(0, 64, 30, b)]


# ------------------------------------------------------------------ facade on the emulation
@pytest.fixture(scope="module")
def env():
    saved = lib_emu_grouped.install()
    cfg = ModelConfig.small()
    yield cfg, synth_all(cfg, seed=0, suppress_stop=False)
    lib_emu_grouped.uninstall(saved)


class _Event:
    def __init__(self, **kw):
        pass

    def record(self):
        pass

    def synchronize(self):
        pass

    def elapsed_time(self, other):
        return 0.0


class _Diffusion:
    """Stands in for DiffusionEngine.sample (a CUDA graph): a deterministic function of every input."""

    def sample(self, lat, cond, iters, noise0, step_noise, cond_free=True, cond_free_k=2.0, pair=None):
        return noise0 + step_noise.sum(0) * 1e-3 + lat.sum() * 1e-4 + cond.sum() * 1e-5 + iters


class _Vocoder:
    def inference(self, mel, z):
        return torch.cat([mel.reshape(-1), z.reshape(-1)])


def _facade(cfg, sds, monkeypatch):
    from tortoise_tts_b200 import api
    from tortoise_tts_b200.ar_engine import AREngine
    from tortoise_tts_b200.clvp_engine import CLVPEngine
    t = api.TextToSpeech.__new__(api.TextToSpeech)
    t.cfg, t.device, t.kv_cache = cfg, torch.device("cpu"), False
    t.enable_redaction = False
    t.debug_capture = False
    t.autoregressive = AREngine(sds["autoregressive"], cfg, device="cpu")
    t.clvp = CLVPEngine(sds["clvp"], cfg, device="cpu")
    t.diffusion, t.vocoder = _Diffusion(), _Vocoder()
    t.cvvp = None
    t.last_timings = {}
    monkeypatch.setattr(api.torch.cuda, "Event", _Event)
    monkeypatch.setattr(api.parallel, "world", lambda: (0, 1))
    # no CUDA graphs on the CPU: the decode loop runs eagerly
    decode = AREngine._decode
    monkeypatch.setattr(AREngine, "_decode", lambda self, st, sp, steps, use_graph, every, tr:
                        decode(self, st, sp, steps, False, every, tr))
    monkeypatch.setattr(AREngine, "MODE", "fused")
    return t


TEXTS = [[42, 2, 194, 91, 24, 2], [7, 77, 8, 9, 100, 12, 13, 14, 15, 3, 2], [5, 6]]
KW = dict(num_autoregressive_samples=3, max_mel_tokens=6, diffusion_iterations=2, use_deterministic_seed=11)


def _cond(cfg):
    g = torch.Generator().manual_seed(3)
    return torch.randn(1, cfg.ar_dim, generator=g), torch.randn(1, 2 * cfg.diff_dim, generator=g)


@pytest.mark.parametrize("k", [1, 2])
def test_tts_batch_equals_one_tts_per_text(env, monkeypatch, k):
    cfg, sds = env
    t = _facade(cfg, sds, monkeypatch)
    calls = []
    gen_grouped = t.autoregressive.generate_grouped
    monkeypatch.setattr(t.autoregressive, "generate_grouped", lambda *a, **kw: calls.append(a[2]) or gen_grouped(*a, **kw))
    cond = _cond(cfg)
    got = t.tts_batch(["a", "b", "c"], preset="ultra_fast", text_tokens_list=TEXTS, conditioning_latents=cond, k=k, **KW)
    assert calls == [[3, 3, 3]], "the three texts must be decoded as one grouped batch"
    assert len(got) == 3
    for u, toks in enumerate(TEXTS):
        want = t.tts_with_preset(None, preset="ultra_fast", text_tokens=toks, conditioning_latents=cond, k=k, **KW)
        if k == 1:
            assert got[u].shape == want.shape and got[u].shape[:2] == (1, 1)
            assert torch.equal(got[u], want)
        else:
            assert isinstance(got[u], list) and len(got[u]) == k == len(want)
            for a, b in zip(got[u], want):
                assert torch.equal(a, b)


def test_grouped_decode_equals_generate(env):
    """generate_grouped: each group's codes and the logits its rows see equal generate() of that utterance alone."""
    from tortoise_tts_b200.ar_engine import AREngine
    cfg, sds = env
    eng = AREngine(sds["autoregressive"], cfg, device="cpu")
    cond = _cond(cfg)[0]
    toks = [t + [0] for t in TEXTS]
    counts = [2, 1, 3]
    torch.manual_seed(4)
    us = [torch.rand(n, 7) for n in counts]
    tr = []
    got = eng.generate_grouped(cond, toks, counts, 7, uniforms_list=us, use_graph=False, trace_logits=tr)
    seen = torch.stack(tr, 1)
    b = 0
    for u, n in enumerate(counts):
        tr1 = []
        want = eng.generate(cond, toks[u], n, 7, uniforms=us[u], use_graph=False, trace_logits=tr1)
        assert torch.equal(got[u], want)
        assert torch.equal(seen[b:b + n], torch.stack(tr1, 1))
        b += n


def test_tts_batch_argument_errors(env, monkeypatch):
    cfg, sds = env
    t = _facade(cfg, sds, monkeypatch)
    with pytest.raises(ValueError):
        t.tts_batch([], preset="ultra_fast")
    with pytest.raises(ValueError):
        t.tts_batch(["a", "b"], preset="ultra_fast", text_tokens_list=[[1, 2]])
    with pytest.raises(TypeError):
        t.tts_batch(["a"], preset="ultra_fast", text_tokens_list=[[1, 2]], no_repeat_ngram_size=2)
    from tortoise_tts_b200 import api
    monkeypatch.setattr(api.parallel, "world", lambda: (0, 2))
    with pytest.raises(NotImplementedError):
        t.tts_batch(["a", "b"], preset="ultra_fast", text_tokens_list=[[1], [2]], k=2)
