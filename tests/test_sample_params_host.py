"""CPU: sampling with per-row settings (ttb_ar_sample_params) — the emulation (tests/lib_emu_params.py) against the scalar
emulations, and the facade with the kernel library replaced by the row-by-row torch emulation: a stream pool whose
streams bring their own settings, chunk size and cross-fade, tts_stream_batch and tts_batch with kwargs_list, and the
argument errors."""
import pytest
import torch

import lib_emu_params
import lib_emu_pool
import lib_emu_typical
from test_fast_batch_host import _fast_facade
from test_stream_pool_host import _rows, _short_streams
from tortoise_tts_b200 import lib
from tortoise_tts_b200.config import ModelConfig
from tortoise_tts_b200.synth import synth_all


@pytest.fixture(scope="module")
def env():
    saved = lib_emu_params.install()
    cfg = ModelConfig.small()
    yield cfg, synth_all(cfg, seed=0, suppress_stop=False)
    lib_emu_params.uninstall(saved)


KW = dict(verbose=False, stream_chunk_size=6)
TEXTS = [[42, 2, 194, 91, 24, 2], [7, 77, 8, 9, 100, 12, 13], [5, 6], [9, 9, 30], [11, 12, 13], [3]]
SETTINGS = [dict(temperature=0.5, top_p=0.9), dict(top_k=3, repetition_penalty=1.4), dict(temperature=1.3, top_k=9),
            dict(top_p=0.4, repetition_penalty=2.7), dict(temperature=0.9, top_k=1), dict(length_penalty=3.0)]


def _state(B, V, N, g):
    seen = torch.zeros(B, (V + 31) // 32, dtype=torch.int32)
    for b in range(B):
        for t in set([1, V - 2] + torch.randint(0, V, (30,), generator=g).tolist()):
            seen[b, t // 32] |= (1 << (t % 32)) if t % 32 < 31 else -(1 << 31)
    return torch.randn(B, V, generator=g) * 3, torch.rand(B, N, generator=g), seen


def test_equal_settings_equal_the_scalar_emulations(env):
    """With the same settings in every row, the per-row emulation gives what lib_emu_pool.ar_sample (with and without
    row_start) and lib_emu_typical.ar_sample_typical give: codes, seen, finished and the counter."""
    cfg, _ = env
    B, V, N = 3, cfg.number_mel_codes, 5
    g = torch.Generator().manual_seed(1)
    logits, u, seen = _state(B, V, N, g)
    rs = torch.tensor([0, 2, -1], dtype=torch.int32)
    sc = dict(temperature=0.7, top_k=9, top_p=0.85, repetition_penalty=1.8)
    args = (0.7, 9, 0.85, 1.8)
    for typical, row_start in ((None, None), (None, rs), (0.6, None)):
        outs = []
        for per_row in (False, True):
            cd, s2, fin = torch.zeros(B, N, dtype=torch.int32), seen.clone(), torch.tensor([0, 1, 0], dtype=torch.int32)
            st = torch.zeros(64, dtype=torch.int32)
            st[0] = 2
            if per_row:
                table = lib.sample_params_table([dict(sc, typical_mass=typical)] * B, "cpu")
                lib_emu_params.ar_sample_params(logits, V, V, B, u, N, s2, cd, N, fin, st, table, cfg.stop_mel_token,
                                                row_start=row_start)
            elif typical is None:
                lib_emu_pool.ar_sample(logits, V, V, B, u, N, s2, cd, N, fin, st, *args, cfg.stop_mel_token,
                                       row_start=row_start)
            else:
                lib_emu_typical.ar_sample_typical(logits, V, V, B, u, N, s2, cd, N, fin, st, *args, cfg.stop_mel_token,
                                                  typical)
            outs.append((cd, s2, fin, st))
        assert all(torch.equal(p, q) for p, q in zip(*outs)), (typical, row_start)


def test_table_words_and_top_k_clamp():
    """The table holds the settings as TtbSampleParams words; the emulation clamps top_k as the kernel does."""
    t = lib.sample_params_table([dict(temperature=0.5, top_k=7, top_p=0.25, repetition_penalty=3.0, typical_mass=0.5),
                                 dict()], "cpu")
    assert t.shape == (2, 8) and t.dtype == torch.int32
    assert t[0, :4].view(torch.float32).tolist() == [0.5, 0.25, 3.0, 0.5] and t[0, 4:].tolist() == [7, 0, 0, 0]
    assert t[1, 3].item() == 0                                           # typical filter off
    t[0, 4], t[1, 4] = 0, 99
    assert [p["top_k"] for p in lib_emu_params.decode_params(t, 2)] == [1, 50]


def test_pool_streams_with_own_settings(env, monkeypatch):
    """Three slots, six texts in three waves, each with its own sampling settings, some with their own chunk size and
    cross-fade: every stream equals the tts_stream emulation of its text with those settings (tokens, chunk count,
    chunk lengths, samples within rounding)."""
    cfg, sds = env
    t = _fast_facade(cfg, sds, monkeypatch)
    _short_streams(monkeypatch)
    ar = t.autoregressive
    ar.w.b_head = ar.w.b_head.clone()
    ar.w.b_head[cfg.stop_mel_token] += 8.0
    per = [dict(s) for s in SETTINGS]
    per[1].update(stream_chunk_size=4, overlap_wav_len=256)
    per[3].update(stream_chunk_size=11)
    per[4].update(overlap_wav_len=2048)
    pool = t.stream_pool(max_streams=3, **KW)
    codes, real_finish = {}, pool._finish

    def finish(s):
        codes[pool.slots[s]["sid"]] = pool.ws.codes()[s, :pool.slots[s]["tokens"]].clone()
        real_finish(s)
    monkeypatch.setattr(pool, "_finish", finish)
    sid_of, out = {}, []
    for wave in ((0, 1), (2, 3), (4, 5)):
        for u in wave:
            sid_of[pool.submit("x", text_tokens=TEXTS[u], use_deterministic_seed=40 + u, **per[u])] = u
        out += pool.poll()
    out += list(pool.run())
    assert pool.ws.sp.get("per_row")
    rows = _rows(out)
    seen = {}
    real_gen = ar.generate_stream

    def gen(*a, **k):
        for y in real_gen(*a, **k):
            seen["codes"] = y[0].clone()
            yield y
    monkeypatch.setattr(ar, "generate_stream", gen)
    for sid, u in sid_of.items():
        want = list(t.tts_stream("x", text_tokens=TEXTS[u], use_deterministic_seed=40 + u, **{**KW, **per[u]}))
        got = rows[sid]
        assert torch.equal(codes[sid], seen["codes"]), "tokens of text %d" % u
        assert [len(c) for c, _ in got] == [len(c) for c in want], "text %d" % u
        assert [last for _, last in got] == [False] * (len(want) - 1) + [True]
        assert max((a - b).abs().max().item() for (a, _), b in zip(got, want)) < 2e-2


def test_pool_stays_on_the_scalar_sampler_with_its_own_settings(env, monkeypatch):
    """Streams that keep the pool's settings (also when given explicitly) never call the per-row sampler; the first
    stream with settings of its own switches the pool to it."""
    cfg, sds = env
    t = _fast_facade(cfg, sds, monkeypatch)
    _short_streams(monkeypatch)
    calls = []
    real = lib.ar_sample_params
    monkeypatch.setattr(lib, "ar_sample_params", lambda *a, **k: calls.append(1) or real(*a, **k))
    pool = t.stream_pool(max_streams=2, temperature=0.7, **KW)
    pool.submit("x", text_tokens=TEXTS[2], use_deterministic_seed=1)
    pool.submit("x", text_tokens=TEXTS[3], use_deterministic_seed=2, temperature=0.7, top_k=50.0)
    out = pool.poll()
    assert not calls and "per_row" not in pool.ws.sp
    pool.submit("x", text_tokens=TEXTS[4], use_deterministic_seed=3, top_p=0.5)
    out += list(pool.run())
    assert calls and pool.ws.sp.get("per_row")
    assert len(_rows(out)) == 3


def test_stream_batch_with_kwargs_list(env, monkeypatch):
    cfg, sds = env
    t = _fast_facade(cfg, sds, monkeypatch)
    _short_streams(monkeypatch)
    out = list(t.tts_stream_batch(["x"] * 4, text_tokens_list=TEXTS[:4], kwargs_list=SETTINGS[:4],
                                  use_deterministic_seed=5, **KW))
    rows = [[c for v, c, _ in out if v == u] for u in range(4)]
    for u in range(4):
        want = list(t.tts_stream("x", text_tokens=TEXTS[u], use_deterministic_seed=5, **KW, **SETTINGS[u]))
        assert [len(c) for c in rows[u]] == [len(c) for c in want], "text %d" % u
        assert max((a - b).abs().max().item() for a, b in zip(rows[u], want)) < 2e-2


def test_tts_batch_with_kwargs_list(env, monkeypatch):
    """Entry u equals tts(texts[u], **kwargs, **kwargs_list[u]), typical sampling included; the long prompt is
    decoded alone with its own settings as scalars."""
    cfg, sds = env
    t = _fast_facade(cfg, sds, monkeypatch)
    texts = TEXTS[:3] + [[5] * 349]
    kl = [dict(SETTINGS[0], typical_sampling=True, typical_mass=0.5), SETTINGS[1], dict(typical_sampling=True),
          dict(SETTINGS[2], typical_sampling=True, typical_mass=0.3)]
    kw = dict(use_deterministic_seed=11, verbose=False, temperature=0.9)
    got = t.tts_batch(["x"] * 4, text_tokens_list=texts, kwargs_list=kl, **kw)
    for u in range(4):
        want = t.tts("x", text_tokens=texts[u], **{**kw, **kl[u]})
        assert torch.equal(got[u], want), "text %d" % u


BAD = [dict(temperature=0.0), dict(temperature=float("nan")), dict(top_k=0), dict(top_k=51), dict(top_k=2.5),
       dict(top_p=0.0), dict(top_p=1.5), dict(repetition_penalty=-1.0), dict(repetition_penalty=float("inf")),
       dict(stream_chunk_size=2.5), dict(overlap_wav_len="x")]


@pytest.mark.parametrize("bad", BAD)
def test_submit_rejects_bad_values_before_queueing(env, monkeypatch, bad):
    cfg, sds = env
    t = _fast_facade(cfg, sds, monkeypatch)
    pool = t.stream_pool(max_streams=1, **KW)
    with pytest.raises(ValueError):
        pool.submit("x", text_tokens=[1, 2], **bad)
    assert not pool._queue and pool._next_sid == 0
    pool.close()


def test_argument_errors(env, monkeypatch):
    cfg, sds = env
    t = _fast_facade(cfg, sds, monkeypatch)
    pool = t.stream_pool(max_streams=1, **KW)
    for key in ("typical_sampling", "no_repeat_ngram_size"):
        with pytest.raises(TypeError):
            pool.submit("x", text_tokens=[1], **{key: True})
    assert not pool._queue
    pool.close()
    with pytest.raises(ValueError):
        t.stream_pool(max_streams=1, top_k=80)
    for call in (t.tts_stream_batch, t.tts_batch):
        with pytest.raises(ValueError):                                   # one dict per text
            call(["a", "b"], text_tokens_list=[[1], [2]], kwargs_list=[{}])
        with pytest.raises(ValueError):
            call(["a"], text_tokens_list=[[1]], kwargs_list=[dict(top_p=2.0)])
        with pytest.raises(TypeError):
            call(["a"], text_tokens_list=[[1]], kwargs_list=[dict(no_repeat_ngram_size=2)])
    with pytest.raises(TypeError):                                        # tts_stream has no typical filter
        t.tts_stream_batch(["a"], text_tokens_list=[[1]], kwargs_list=[dict(typical_sampling=True)])
    with pytest.raises(ValueError):
        t.tts_batch(["a"], text_tokens_list=[[1]], kwargs_list=[dict(typical_sampling=True, typical_mass=0.0)])
