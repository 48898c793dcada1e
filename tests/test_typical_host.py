"""CPU: typical sampling (the reference's `typical_sampling` / `typical_mass` tts kwargs) through the engine and both
facades, with the kernel library replaced by the torch emulation (tests/lib_emu.py + tests/lib_emu_typical.py). The
kernel itself is checked on the GPU by tests/test_gpu_typical.py."""
import contextlib
import dataclasses

import pytest
import torch

import lib_emu_typical
import typical_oracle
from tortoise_tts_b200.config import ModelConfig
from tortoise_tts_b200.synth import synth_all

TEXT = [12, 40, 7, 99, 3]


@pytest.fixture(scope="module")
def env():
    saved = lib_emu_typical.install()
    cfg = ModelConfig.small()
    yield cfg, synth_all(cfg, seed=0, suppress_stop=False)
    lib_emu_typical.uninstall(saved)


@pytest.fixture
def calls(monkeypatch):
    """Records every sampler call: (entry name, positional args, keyword args)."""
    import tortoise_tts_b200.lib as lib
    log = []
    for name in ("ar_sample", "ar_sample_typical"):
        fn = getattr(lib, name)

        def rec(*a, _fn=fn, _name=name, **k):
            log.append((_name, a, k))
            return _fn(*a, **k)
        monkeypatch.setattr(lib, name, rec)
    return log


def _engine(cfg, sds, monkeypatch, mode, chains):
    from tortoise_tts_b200.ar_engine import AREngine
    monkeypatch.setattr(AREngine, "MODE", mode)
    monkeypatch.setattr(AREngine, "FUSED_MAX_B", 64)
    monkeypatch.setattr(AREngine, "CHAINS", chains)
    monkeypatch.setattr(AREngine, "CHAINS_MIN_B", 2)
    return AREngine(sds["autoregressive"], cfg, device="cpu")


@pytest.mark.parametrize("mode,chains", [("fused", 1), ("mixed", 1), ("mixed", 2), ("perop", 1)])
def test_every_sample_site_takes_the_typical_entry(env, monkeypatch, calls, mode, chains):
    cfg, sds = env
    eng = _engine(cfg, sds, monkeypatch, mode, chains)
    u = torch.rand(4, 5, generator=torch.Generator().manual_seed(1))
    cond = torch.randn(cfg.ar_dim, generator=torch.Generator().manual_seed(2))
    eng.generate(cond, TEXT, 4, 5, uniforms=u, use_graph=False, typical_mass=0.7)
    st = eng._dec
    assert st["mode"] == ("perop" if mode == "perop" else mode) and len(st["chains"]) == chains
    names = [c[0] for c in calls]
    assert names == ["ar_sample_typical"] * (5 * chains)
    # the prefill's first sample broadcasts row 0 of the prompt logits (ld_logits = 0), the decode steps read their rows
    assert [c[1][1] for c in calls[:chains]] == [0] * chains
    assert all(c[1][1] == cfg.number_mel_codes for c in calls[chains:])
    assert all(c[1][-1] == pytest.approx(0.7) for c in calls)


@pytest.mark.parametrize("mode,chains", [("fused", 1), ("mixed", 2), ("perop", 1)])
def test_filter_off_keeps_the_old_call(env, monkeypatch, calls, mode, chains):
    cfg, sds = env
    eng = _engine(cfg, sds, monkeypatch, mode, chains)
    u = torch.rand(4, 4, generator=torch.Generator().manual_seed(3))
    cond = torch.randn(cfg.ar_dim, generator=torch.Generator().manual_seed(4))
    eng.generate(cond, TEXT, 4, 4, uniforms=u, use_graph=False)
    assert [c[0] for c in calls] == ["ar_sample"] * (4 * chains)
    for name, a, k in calls:
        # logits, ld, V, B, uniforms, ld_u, seen, codes, ld_codes, finished, state, T, top_k, top_p, rep, stop
        assert len(a) == 16 and k == {"advance": True}
        assert a[2] == cfg.number_mel_codes and a[3] == 4 // chains and a[5] == a[8] == 4
        assert a[11:] == (0.8, 50, 0.8, 2.0, cfg.stop_mel_token)


def test_two_chains_match_one_chain(env, monkeypatch):
    cfg, sds = env
    u = torch.rand(4, 7, generator=torch.Generator().manual_seed(5))
    cond = torch.randn(cfg.ar_dim, generator=torch.Generator().manual_seed(6))
    outs = []
    for n in (1, 2):
        eng = _engine(cfg, sds, monkeypatch, "mixed", n)
        outs.append(eng.generate(cond, TEXT, 4, 7, uniforms=u, use_graph=False, typical_mass=0.6))
        assert len(eng._dec["chains"]) == n
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("mass", [0.3, 0.9])
def test_engine_decode_against_oracle(env, mass):
    """Every token the engine draws lies in the oracle's kept set (tests/typical_oracle.py) for the logits of its own
    sequence and the same uniform. (The untrained synthetic model is nearly flat, so T holds thousands of tokens and the
    emulated bf16 trunk, rounding differently from the oracle's fp32 one, reorders them: the drawn token itself is
    compared on the GPU, on the kernel.)"""
    from tortoise_tts_b200.ar_engine import AREngine
    from oracle import ar
    cfg, sds = env
    eng = AREngine(sds["autoregressive"], cfg, device="cpu")
    u = torch.rand(3, 6, generator=torch.Generator().manual_seed(7))
    cond = torch.randn(cfg.ar_dim, generator=torch.Generator().manual_seed(8))
    codes = eng.generate(cond, TEXT, 3, 6, uniforms=u, use_graph=False, typical_mass=mass).long()
    with torch.no_grad():
        lg = ar.teacher_forced_logits(sds["autoregressive"], cfg, cond, TEXT, codes[:, :-1], "ref_kv_quirk")
    for b in range(3):
        seen = {1, cfg.start_mel_token}
        for n in range(6):
            if n > 0 and int(codes[b, n - 1]) == cfg.stop_mel_token:
                assert int(codes[b, n]) == cfg.stop_mel_token
                continue
            _, kept, _ = typical_oracle.sample_step(lg[b, n], seen, float(u[b, n]), typical_mass=mass)
            assert int(codes[b, n]) in kept.tolist()
            seen.add(int(codes[b, n]))


def test_out_of_range_mass_raises(env):
    from tortoise_tts_b200.ar_engine import AREngine
    from tortoise_tts_b200 import api
    cfg, sds = env
    eng = AREngine(sds["autoregressive"], cfg, device="cpu")
    for m in (0.0, -0.1, 1.5, float("nan")):
        with pytest.raises(ValueError):
            eng.generate(torch.zeros(cfg.ar_dim), TEXT, 2, 3, use_graph=False, typical_mass=m)
        with pytest.raises(ValueError):
            api._typical_mass(True, m)
    assert api._typical_mass(False, 5.0) is None
    assert api._typical_mass(True, 1.0) == 1.0


class _Reached(Exception):
    pass


class _Event:
    def __init__(self, *a, **k):
        pass

    def record(self):
        pass


def _api_facade(cfg, monkeypatch, log):
    """api.TextToSpeech whose AR engine records its kwargs and stops the call (the rest of tts() needs a GPU)."""
    from tortoise_tts_b200 import api

    class _AR:
        def generate(self, *a, **k):
            log.append(k)
            raise _Reached()
    t = api.TextToSpeech.__new__(api.TextToSpeech)
    t.cfg, t.device, t.kv_cache = cfg, torch.device("cpu"), True
    t.autoregressive = _AR()
    monkeypatch.setattr(api.torch.cuda, "Event", _Event)
    monkeypatch.setattr(api.parallel, "world", lambda: (0, 1))
    return t


def test_api_tts_paths_pass_the_mass(env, monkeypatch):
    cfg, _ = env
    log = []
    t = _api_facade(cfg, monkeypatch, log)
    lat = (torch.zeros(cfg.ar_dim), torch.zeros(cfg.ar_dim))
    kw = dict(conditioning_latents=lat, text_tokens=TEXT, use_deterministic_seed=1, num_autoregressive_samples=2,
              max_mel_tokens=4)
    with pytest.raises(_Reached):
        t.tts("x", **kw)
    with pytest.raises(_Reached):
        t.tts("x", typical_sampling=True, **kw)
    with pytest.raises(_Reached):
        t.tts("x", typical_sampling=True, typical_mass=0.25, **kw)
    with pytest.raises(_Reached):
        t.tts_with_preset("x", preset="ultra_fast", typical_sampling=True, typical_mass=0.5, **kw)
    with pytest.raises(_Reached):
        t.tts_long("x", preset="ultra_fast", text_tokens_list=[TEXT], typical_sampling=True, typical_mass=0.4,
                   **{k: v for k, v in kw.items() if k != "text_tokens"})
    assert [k["typical_mass"] for k in log] == [None, 0.9, 0.25, 0.5, 0.4]
    with pytest.raises(ValueError):
        t.tts("x", typical_sampling=True, typical_mass=0.0, **kw)
    with pytest.raises(TypeError):
        t.tts("x", typical_p=0.5, **kw)


def test_api_fast_tts_and_stream(env, monkeypatch, calls):
    """api_fast.tts samples through the typical entry; tts_stream rejects the kwargs, as the reference's streaming
    generator has no such parameter (autoregressive.py:565-574)."""
    from tortoise_tts_b200 import api_fast
    from tortoise_tts_b200.ar_engine import AREngine
    from tortoise_tts_b200.hifigan_engine import HifiganEngine
    cfg, sds = env
    t = api_fast.TextToSpeech.__new__(api_fast.TextToSpeech)
    t.cfg, t.device, t.kv_cache, t._sds = cfg, torch.device("cpu"), True, sds
    t.autoregressive = AREngine(sds["autoregressive"], cfg, device="cpu")
    t.hifi_decoder = HifiganEngine(sds["hifigan"], cfg, device="cpu")
    t.rlg_auto = t._conditioning = t._tokenizer = None
    t.models_dir = None
    t.last_timings = {}
    voice = torch.randn(1, cfg.ar_dim, generator=torch.Generator().manual_seed(9))
    monkeypatch.setattr(t, "get_random_conditioning_latents", lambda: voice)
    t.cfg = dataclasses.replace(cfg, max_mel_tokens=6)
    wav = t.tts("x", text_tokens=TEXT, use_deterministic_seed=3, verbose=False, typical_sampling=True, typical_mass=0.5)
    assert wav.dim() == 3 and calls and all(c[0] == "ar_sample_typical" and c[1][-1] == 0.5 for c in calls)
    n = len(calls)
    t.tts("x", text_tokens=TEXT, use_deterministic_seed=3, verbose=False)
    assert all(c[0] == "ar_sample" for c in calls[n:])
    for kw in (dict(typical_sampling=True), dict(typical_mass=0.5)):
        with pytest.raises(TypeError):
            next(t.tts_stream("x", text_tokens=TEXT, verbose=False, **kw))
    with pytest.raises(TypeError):
        t.tts("x", text_tokens=TEXT, verbose=False, typical_p=0.5)


def test_graph_recaptured_when_mass_changes(env, monkeypatch):
    """The captured decode step is keyed on the sampling parameters: a new typical_mass (or switching the filter on
    or off) captures a new graph, the same one replays the old graph. CUDA graph capture is stubbed out here."""
    from tortoise_tts_b200.ar_engine import AREngine
    cfg, sds = env
    captured = []

    class _Graph:
        def __init__(self):
            captured.append(self)

        def replay(self):
            pass

    class _Stream:
        def __init__(self, *a, **k):
            pass

        def wait_stream(self, s):
            pass
    monkeypatch.setattr(torch.cuda, "CUDAGraph", _Graph)
    monkeypatch.setattr(torch.cuda, "Stream", _Stream)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: _Stream())
    monkeypatch.setattr(torch.cuda, "stream", lambda s: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "graph", lambda g, stream=None: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a: None)
    eng = _engine(cfg, sds, monkeypatch, "mixed", 1)
    cond = torch.zeros(cfg.ar_dim)
    seen_params = []
    for m in (0.5, 0.5, 0.8, None, None, 0.8):
        eng.generate(cond, TEXT, 2, 3, seed=0, typical_mass=m)
        seen_params.append(eng._dec["graph_params"].get("typical_mass"))
    assert seen_params == [0.5, 0.5, 0.8, None, None, 0.8]
    assert len(captured) == 4          # 0.5, 0.8, off, 0.8 again
