"""CPU: the stream pool of the api_fast path (continuous batching) — per-row start steps in the emulated kernels,
AREngine.slot_workspace, and TextToSpeech.stream_pool against tts_stream per text, with the kernel library replaced by
the row-by-row torch emulation (tests/lib_emu.py + lib_emu_grouped.py + lib_emu_stream.py + lib_emu_pool.py)."""
import threading

import pytest
import torch

import lib_emu_pool
from test_fast_batch_host import _fast_facade
from tortoise_tts_b200 import api_fast
from tortoise_tts_b200.api_fast import stream_flushes
from tortoise_tts_b200.config import ModelConfig
from tortoise_tts_b200.synth import synth_all


@pytest.fixture(scope="module")
def env():
    saved = lib_emu_pool.install()
    cfg = ModelConfig.small()
    yield cfg, synth_all(cfg, seed=0, suppress_stop=False)
    lib_emu_pool.uninstall(saved)


KW = dict(verbose=False, stream_chunk_size=6)


def _short_streams(monkeypatch):
    """Streams of at most 40 - P tokens with a first flush at 10 tokens, so that the emulation runs in seconds."""
    monkeypatch.setattr(api_fast, "STREAM_MAX_LENGTH", 40)
    monkeypatch.setattr(api_fast, "FIRST_BUFFER", 10)


def test_row_start_none_and_zero_equal_the_stream_emulation(env):
    """row_start=None is the existing emulation, and all-zero start steps give the same numbers."""
    import lib_emu
    import lib_emu_stream
    cfg, _ = env
    g = torch.Generator().manual_seed(0)
    B, D, V, N = 3, cfg.ar_dim, cfg.number_mel_codes, 7
    emb, pos = torch.randn(V, D, generator=g), torch.randn(N + 2, D, generator=g)
    codes = torch.randint(0, V, (B, N), generator=g, dtype=torch.int32)
    st = torch.zeros(64, dtype=torch.int32)
    st[0] = 4
    zeros = torch.zeros(B, dtype=torch.int32)
    a, b, c = (torch.empty(B, D) for _ in range(3))
    lib_emu.ar_embed_step(codes, N, st, emb, pos, B, D, 1, a)
    lib_emu_pool.ar_embed_step(codes, N, st, emb, pos, B, D, 1, b)
    lib_emu_pool.ar_embed_step(codes, N, st, emb, pos, B, D, 1, c, row_start=zeros)
    assert torch.equal(a, b) and torch.equal(a, c)
    x = torch.randn(B, D, generator=g)
    gg, bb = torch.ones(D), torch.zeros(D)
    o1, o2 = torch.zeros(B, N, D), torch.zeros(B, N, D)
    lib_emu_stream.ar_capture_latents(x, B, D, gg, bb, gg, bb, st, N, o1, N * D)
    lib_emu_pool.ar_capture_latents(x, B, D, gg, bb, gg, bb, st, N, o2, N * D, row_start=zeros)
    assert torch.equal(o1, o2)
    logits = torch.randn(B, V, generator=g)
    u = torch.rand(B, N, generator=g)
    outs = []
    for rs in (None, zeros):
        seen = torch.zeros(B, (V + 31) // 32, dtype=torch.int32)
        cd, fin, s2 = codes.clone(), torch.zeros(B, dtype=torch.int32), st.clone()
        lib_emu_pool.ar_sample(logits, V, V, B, u, N, seen, cd, N, fin, s2, 0.8, 50, 0.8, 2.0, cfg.stop_mel_token,
                               row_start=rs)
        outs.append((cd, seen, fin, s2))
    assert all(torch.equal(p, q) for p, q in zip(*outs))


def test_idle_rows_stay_inside_their_rows(env):
    """A row whose start lies 1000 steps back (or ahead) is clamped: every index stays in [0, Nmax)."""
    cfg, _ = env
    B, D, V, N = 2, cfg.ar_dim, cfg.number_mel_codes, 5
    emb, pos = torch.randn(V, D), torch.randn(N + 2, D)
    codes = torch.zeros(B, N, dtype=torch.int32)
    st = torch.zeros(64, dtype=torch.int32)
    st[0] = 3
    rs = torch.tensor([-1000, 1000], dtype=torch.int32)
    x = torch.empty(B, D)
    lib_emu_pool.ar_embed_step(codes, N, st, emb, pos, B, D, 1, x, row_start=rs)
    assert torch.equal(x[0], emb[0] + pos[N + 1]) and torch.equal(x[1], emb[0] + pos[2])
    fin = torch.tensor([1, 1], dtype=torch.int32)
    lib_emu_pool.ar_sample(torch.zeros(B, V), V, V, B, torch.rand(B, N), N, torch.zeros(B, 256, dtype=torch.int32),
                           codes, N, fin, st, 0.8, 50, 0.8, 2.0, 7, row_start=rs)
    assert codes[0].tolist() == [0, 0, 0, 0, 7] and codes[1].tolist() == [7, 0, 0, 0, 0] and int(st[0]) == 4
    out = torch.zeros(B, N, D)
    lib_emu_pool.ar_capture_latents(torch.randn(B, D), B, D, torch.ones(D), torch.zeros(D), torch.ones(D),
                                    torch.zeros(D), st, N, out, N * D, row_start=rs)
    assert out.abs().sum().item() == 0.0


def _rows(out):
    rows = {}
    for sid, chunk, last in out:
        assert not rows.get(sid) or not rows[sid][-1][1], "a chunk after the last one of stream %d" % sid
        rows.setdefault(sid, []).append((chunk, last))
    return rows


def _flush_counts(t, monkeypatch):
    """Wraps the HiFiGAN batch call to record the token count of every flush of every stream."""
    seen = []
    real = t.hifi_decoder.inference_batch

    def wrapped(lat, spk):
        seen.append((int(lat.shape[0]), int(lat.shape[1])))
        return real(lat, spk)
    monkeypatch.setattr(t.hifi_decoder, "inference_batch", wrapped)
    return seen


TEXTS = [[42, 2, 194, 91, 24, 2], [7, 77, 8, 9, 100, 12, 13, 14, 15, 3, 2], [5, 6], [9, 9, 30], [11, 12, 13],
         [3], [60, 61, 62, 63, 64, 65, 66, 67, 68, 69, 70, 71, 72, 73, 74, 75, 76], [8, 8], [99, 98, 97, 96]]


def test_pool_streams_equal_tts_stream_in_waves(env, monkeypatch):
    """Three slots, nine texts with their own seeds and two voices, in three waves submitted between polls (one wave
    from another thread): every stream's chunks have tts_stream's count, lengths and `last` flags, and its samples
    agree within rounding; a slot is reused three times; one slot idles for more than Nmax global steps; rows end by
    their stop token and by their cap."""
    cfg, sds = env
    t = _fast_facade(cfg, sds, monkeypatch)
    _short_streams(monkeypatch)
    g = torch.Generator().manual_seed(5)
    voices = [t.get_random_conditioning_latents(), torch.randn(1, cfg.ar_dim, generator=g)]
    ar = t.autoregressive                 # a stop logit raised so that some rows stop (one at its very first token)
    ar.w.b_head = ar.w.b_head.clone()
    ar.w.b_head[cfg.stop_mel_token] += 8.0
    pool = t.stream_pool(max_streams=3, **KW)
    ws = pool.ws
    admits, real_admit = [], ws.admit

    def admit(slot, *a):
        admits.append((slot, ws.step))
        return real_admit(slot, *a)
    monkeypatch.setattr(ws, "admit", admit)
    sub = {}

    def submit(u):
        sub[pool.submit("x", conditioning_latent=voices[u % 2], text_tokens=TEXTS[u], use_deterministic_seed=20 + u)] = u
    # one text at a time while at most two slots are busy (the lowest free slot is taken first, so slot 2 idles for more
    # than Nmax global steps), then the rest at once from another thread
    order, out = iter(range(9)), []
    while ws.step <= api_fast.STREAM_MAX_LENGTH + 5:
        if sum(r is not None for r in pool.slots) < 2 and not pool._queue:
            submit(next(order))
        out += pool.poll()
    th = threading.Thread(target=lambda: [submit(u) for u in order])
    th.start()
    th.join()
    out += list(pool.run())
    assert pool.poll() == []
    rows = _rows(out)
    assert sorted(sub.values()) == list(range(9)) and set(rows) == set(sub)
    uses = [s for s, _ in admits]
    assert max(uses.count(s) for s in range(3)) >= 3, uses
    assert [st for s, st in admits if s == 2][0] > api_fast.STREAM_MAX_LENGTH, admits
    kinds = set()
    for sid, u in sub.items():
        monkeypatch.setattr(t, "_auto_latent", lambda v, u=u: voices[u % 2].reshape(-1))
        want = list(t.tts_stream("x", text_tokens=TEXTS[u], use_deterministic_seed=20 + u, **KW))
        got = rows[sid]
        assert [len(c) for c, _ in got] == [len(c) for c in want], "stream %d" % u
        assert [last for _, last in got] == [False] * (len(want) - 1) + [True]
        assert max((a - b).abs().max().item() for (a, _), b in zip(got, want)) < 2e-2
        n, cap = pool.last_timings[sid]["tokens"], 40 - (len(TEXTS[u]) + 5)
        kinds.add("cap" if n == cap else "stop")
        tim = pool.last_timings[sid]
        assert 0.0 <= tim["wait_admit_s"] <= tim["wait_first_chunk_s"]
    assert kinds == {"cap", "stop"}, kinds


def test_flushes_follow_the_rule_whatever_the_admission_step(env, monkeypatch):
    """The token counts HiFiGAN sees for a stream are its stream_flushes sequence, however late it was admitted."""
    cfg, sds = env
    t = _fast_facade(cfg, sds, monkeypatch)
    _short_streams(monkeypatch)
    calls = _flush_counts(t, monkeypatch)
    pool = t.stream_pool(max_streams=2, **KW)
    a = pool.submit("x", text_tokens=TEXTS[3], use_deterministic_seed=1)
    out = pool.poll()
    b = pool.submit("x", text_tokens=TEXTS[3], use_deterministic_seed=1)      # same text and seed, admitted later
    out += list(pool.run())
    rows = _rows(out)
    assert [len(c) for c, _ in rows[a]] == [len(c) for c, _ in rows[b]]
    n = pool.last_timings[a]["tokens"]
    assert n == pool.last_timings[b]["tokens"]
    cap = 40 - (len(TEXTS[3]) + 5)
    stop_at = n if n < cap else None
    want, flushed, target = [], 0, 10
    while True:                                    # the yields of generate_stream, as tts_stream flushes them
        have = min(target, cap)
        m, ended = (stop_at, True) if stop_at is not None and stop_at <= have else (have, have >= cap)
        for _ in stream_flushes(m, flushed, ended, 6):
            want.append(m)
            flushed = m
        if ended:
            break
        target = have + 6
    counts = [L for R, L in calls for _ in range(R)]
    assert sorted(counts) == sorted(want + want)


def test_pool_argument_errors(env, monkeypatch):
    cfg, sds = env
    t = _fast_facade(cfg, sds, monkeypatch)
    from tortoise_tts_b200 import lib
    from tortoise_tts_b200.ar_engine import AREngine
    for bad in (0, 257):
        with pytest.raises(ValueError):
            t.stream_pool(max_streams=bad)
    with pytest.raises(TypeError):
        t.stream_pool(max_streams=2, no_repeat_ngram_size=2)
    with pytest.raises(TypeError):
        t.stream_pool(max_streams=2, typical_sampling=True)
    pool = t.stream_pool(max_streams=1, **KW)
    with pytest.raises(ValueError):                                      # P = 349 + 1 + 4 = 354 > 352
        pool.submit("a", text_tokens=[5] * 349)
    pool.submit("a", text_tokens=[5] * 347)                             # P = 352 is accepted
    with pytest.raises(ValueError):
        pool.submit("a", voice_samples=["clip"], conditioning_latent=torch.zeros(1, cfg.ar_dim), text_tokens=[1])
    pool.close()
    with pytest.raises(RuntimeError):
        pool.submit("a", text_tokens=[1])
    monkeypatch.setattr(AREngine, "MODE", "perop")
    with pytest.raises(lib.TtbError):
        t.stream_pool(max_streams=2)
