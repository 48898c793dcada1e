"""GPU: the per-row sampler (ttb_ar_sample_params, include/ttb.h TtbSampleParams) — against the scalar entries with equal
settings and row by row with mixed settings, in the slot workspace's three step forms, and through the facade: the stream
pool, tts_stream_batch and tts_batch with per-text settings against the per-text calls."""
import pytest
import torch

from gpu_util import report
from test_gpu_stream_pool import WAVE_ABS, _mode, _one_warp_mixed, fast, medium  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

V = 8194
STOP = 8193


def _inputs(B, N, seed):
    g = torch.Generator().manual_seed(seed)
    logits = (torch.randn(B, V, generator=g) * torch.linspace(0.5, 6.0, B).unsqueeze(1)).cuda()
    u = torch.rand(B, N, generator=g).cuda()
    seen = torch.zeros(B, (V + 31) // 32, dtype=torch.int32)
    for b in range(B):
        for t in set([1, 8192] + torch.randint(0, 8192, (20,), generator=g).tolist()):
            seen[b, t // 32] |= (1 << (t % 32)) if t % 32 < 31 else -(1 << 31)
    return logits, u, seen.cuda()


def _run(fn, B, N, seen, fin, step=0):
    """(codes, seen, finished, state) after one call of fn(codes, seen, finished, state)."""
    codes = torch.full((B, N), -1, dtype=torch.int32, device="cuda")
    s, f = seen.clone(), fin.clone()
    state = torch.zeros(64, dtype=torch.int32, device="cuda")
    state[0] = step
    fn(codes, s, f, state)
    torch.cuda.synchronize()
    return codes, s, f, state


def _same(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("B", [1, 5, 256])
@pytest.mark.parametrize("advance", [True, False])
def test_equal_settings_equal_the_scalar_entries(B, advance):
    """Every row with the same settings: ttb_ar_sample_params gives ttb_ar_sample's, ttb_ar_sample_rows' (row_start)
    and ttb_ar_sample_typical's codes, seen, finished and state bit for bit, with finished rows among them."""
    from tortoise_tts_b200 import lib
    N = 6
    logits, u, seen = _inputs(B, N, B)
    fin = torch.zeros(B, dtype=torch.int32, device="cuda")
    fin[B // 2] = 1 if B > 1 else 0
    rs = torch.tensor([(3 * b) % 5 - 2 for b in range(B)], dtype=torch.int32, device="cuda")
    sc = (0.8, 50, 0.8, 2.0)
    base = dict(temperature=0.8, top_k=50, top_p=0.8, repetition_penalty=2.0)

    def scalar(c, s, f, st):
        lib.ar_sample(logits, V, V, B, u, N, s, c, N, f, st, *sc, STOP, advance=advance)

    def rows(c, s, f, st):
        lib.ar_sample(logits, V, V, B, u, N, s, c, N, f, st, *sc, STOP, advance=advance, row_start=rs)

    def typical(c, s, f, st):
        lib.ar_sample_typical(logits, V, V, B, u, N, s, c, N, f, st, *sc, STOP, 0.9, advance=advance)

    for ref, extra, kw in ((scalar, {}, {}), (rows, {}, {"row_start": rs}), (typical, {"typical_mass": 0.9}, {})):
        table = lib.sample_params_table([{**base, **extra}] * B, "cuda")

        def per_row(c, s, f, st):
            lib.ar_sample_params(logits, V, V, B, u, N, s, c, N, f, st, table, STOP, advance=advance, **kw)
        for step in (0, 3):
            assert _same(_run(ref, B, N, seen, fin, step), _run(per_row, B, N, seen, fin, step)), (ref.__name__, step)


def _mixed_rows(B, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for b in range(B):
        r = dict(temperature=[0.3, 0.8, 1.5][b % 3], top_k=[1, 7, 50][(b // 3) % 3],
                 top_p=[0.05, 0.5, 1.0, 0.8][(b // 9) % 4], repetition_penalty=1.0 + 2.0 * torch.rand(1, generator=g).item())
        m = [None, 0.2, 0.9, 1.0][b % 4]
        if m is not None:
            r["typical_mass"] = m
        out.append(r)
    return out


def test_mixed_settings_row_by_row():
    """256 rows with their own temperature (0.3-1.5), top_k (1, 7, 50), top_p (0.05-1.0), repetition penalty (1-3) and
    typical filter (off, 0.2, 0.9, 1.0), some with row_start: row b equals the scalar kernel on row b alone with its
    settings bit for bit, and its token agrees with the float64 oracle up to rounding boundaries."""
    from tortoise_tts_b200 import lib
    from oracle.ar import sample_step
    import typical_oracle
    B, N = 256, 4
    logits, u, seen = _inputs(B, N, 11)
    fin = torch.zeros(B, dtype=torch.int32, device="cuda")
    fin[17] = 1
    rows = _mixed_rows(B, 2)
    table = lib.sample_params_table(rows, "cuda")
    rs = torch.tensor([b % 3 - 1 for b in range(B)], dtype=torch.int32, device="cuda")
    step = 2
    got = _run(lambda c, s, f, st: lib.ar_sample_params(logits, V, V, B, u, N, s, c, N, f, st, table, STOP,
                                                         row_start=rs), B, N, seen, fin, step)
    mism = 0
    for b in range(B):
        r = rows[b]
        col = step - int(rs[b])
        sc = (r["temperature"], r["top_k"], r["top_p"], r["repetition_penalty"])
        lg, uu = logits[b:b + 1], u[b:b + 1].clone()

        def one(c, s, f, st):
            if "typical_mass" in r:
                lib.ar_sample_typical(lg, V, V, 1, uu, N, s, c, N, f, st, *sc, STOP, r["typical_mass"])
            else:
                lib.ar_sample(lg, V, V, 1, uu, N, s, c, N, f, st, *sc, STOP)
        want = _run(one, 1, N, seen[b:b + 1], fin[b:b + 1], col)
        assert torch.equal(got[0][b], want[0][0]) and torch.equal(got[1][b], want[1][0]), "row %d" % b
        assert torch.equal(got[2][b], want[2][0]), "row %d" % b
        if b == 17:
            assert int(got[0][b, col]) == STOP
            continue
        prev = [w * 32 + bit for w in range(seen.shape[1]) for bit in range(32) if (int(seen[b, w]) >> bit) & 1]
        lrow, ub = logits[b].cpu(), float(u[b, col])
        if "typical_mass" in r:
            tok, kept, _ = typical_oracle.sample_step(lrow, prev, ub, *sc, r["typical_mass"])
        else:
            tok, kept, _ = sample_step(lrow, prev, ub, *sc)
        t = int(got[0][b, col])
        if t != tok:
            mism += 1
            assert t in [int(k) for k in kept] or "typical_mass" in r, (b, t, tok)
    assert int(got[3][0]) == step + 1
    report("per-row sampler vs float64 oracle: mismatching rows of 256", mism)
    assert mism <= 4


@pytest.mark.parametrize("mode,C", [("fused", 4), ("mixed", 24), ("mixed", 128)])
def test_slot_rows_with_own_settings(medium, mode, C):
    """Rows with different settings admitted at different steps give the codes and latents that the same rows give in a
    workspace where every row has its settings from step 0 (at 128 slots the copies run in other decode chains). A row
    with the workspace's settings runs on the scalar sampler until the first row with its own settings switches the
    step to the per-row sampler, and keeps its tokens across the switch; after the switch, rows with new settings join
    without a new step graph."""
    cfg, eng = medium
    g = torch.Generator().manual_seed(8)
    toks = [torch.randint(1, 255, (n,), generator=g).tolist() + [0] for n in (30, 120, 9)]
    voices = [torch.randn(cfg.ar_dim, generator=g).cuda() for _ in toks]
    N = 120
    us = [torch.rand(N, generator=g).cuda() for _ in toks]
    sets = [dict(temperature=0.5, top_k=7, top_p=0.9, repetition_penalty=1.3),
            dict(temperature=1.4, top_k=50, top_p=1.0, repetition_penalty=2.8),
            dict(temperature=0.9, top_k=1, top_p=0.3)]
    restore = _mode(mode)
    try:
        ref = eng.slot_workspace(C, N)
        for i in range(3):
            ref.admit(i, voices[i], toks[i], us[i], sets[i])
        ref.admit(3, voices[2], toks[2], us[2])                    # the workspace's settings, per-row sampler
        ref.advance(90)
        ref.check()
        rc, rl, rn = ref.codes().clone(), ref.latents.clone(), [ref.tokens(i) for i in range(4)]
        del ref
        ws = eng.slot_workspace(C, N)
        scalar_graph = ws.st["graph"]
        ws.admit(0, voices[2], toks[2], us[2], dict(temperature=0.8))   # equal to the defaults: stays scalar
        ws.advance(5)
        assert "per_row" not in ws.sp and ws.st["graph"] is scalar_graph
        slots = [C - 1, C // 2, 1]
        ws.admit(slots[0], voices[0], toks[0], us[0], sets[0])
        assert ws.sp.get("per_row") and ws.st["graph"] is not scalar_graph
        graph = ws.st["graph"]
        ws.advance(11)
        ws.admit(slots[1], voices[1], toks[1], us[1], sets[1])
        ws.advance(23)
        ws.admit(slots[2], voices[2], toks[2], us[2], sets[2])
        ws.advance(60)
        ws.check()
        assert ws.st["graph"] is graph
        codes, lat = ws.codes(), ws.latents
        for i, s in enumerate(slots + [0]):
            n = min(ws.tokens(s), rn[i])
            assert torch.equal(codes[s, :n], rc[i, :n]), "codes of row %d" % i
            assert torch.equal(lat[s, :n], rl[i, :n]), "latents of row %d" % i
    finally:
        restore()


SETTINGS = [dict(temperature=0.6, top_p=0.9), dict(top_k=7, repetition_penalty=1.5), dict(temperature=1.2, top_k=20),
            dict(top_p=0.5, repetition_penalty=3.0), dict(temperature=0.4, top_k=3, top_p=1.0), dict(length_penalty=2.0)]


def test_pool_streams_with_own_settings(fast):
    """8 slots, 12 texts over two voices and 12 seeds in three waves, each with its own settings and some with their own
    chunk size and cross-fade (mixed step, one warp per stream): every stream gives tts_stream's tokens bit for bit with
    those settings, its chunk count and lengths, and samples within WAVE_ABS."""
    from test_gpu_stream_batch import _recorded_codes
    tts, cfg, clips, voices = fast
    g = torch.Generator().manual_seed(12)
    lens = torch.randint(5, 60, (12,), generator=g).tolist()
    toks = [torch.randint(1, 255, (n,), generator=g).tolist() for n in lens]
    which = [u % 2 for u in range(12)]
    per = [dict(SETTINGS[u % len(SETTINGS)]) for u in range(12)]
    per[1].update(stream_chunk_size=25, overlap_wav_len=512)
    per[6].update(stream_chunk_size=60)
    per[9].update(overlap_wav_len=2048)
    restore = _one_warp_mixed()
    try:
        pool = tts.stream_pool(max_streams=8, verbose=False)
        graph = None
        codes = {}
        real_finish = pool._finish

        def finish(s):
            codes[pool.slots[s]["sid"]] = pool.ws.codes()[s, :pool.slots[s]["tokens"]].clone()
            real_finish(s)
        pool._finish = finish
        sid_of, out = {}, []
        for wave in ((0, 1, 2, 3, 4), (5, 6, 7, 8), (9, 10, 11)):
            for u in wave:
                sid_of[pool.submit("x", voice_samples=clips[which[u]], text_tokens=toks[u],
                                   use_deterministic_seed=30 + u, **per[u])] = u
            for _ in range(3):
                out += pool.poll()
            graph = graph or pool.ws.st["graph"]                  # the per-row graph, captured at the first admission
        out += list(pool.run())
        assert pool.ws.sp.get("per_row") and pool.ws.st["graph"] is graph
        box, unwrap = _recorded_codes(tts, "generate_stream")
        worst = 0.0
        for sid, u in sid_of.items():
            got = [c for v, c, _ in out if v == sid]
            want = list(tts.tts_stream("x", voice_samples=clips[which[u]], text_tokens=toks[u],
                                       use_deterministic_seed=30 + u, verbose=False, **per[u]))
            assert torch.equal(codes[sid], box["codes"]), "tokens of text %d" % u
            assert [len(c) for c in got] == [len(c) for c in want], "chunks of text %d" % u
            worst = max(worst, max((a - b).abs().max().item() for a, b in zip(got, want) if a.numel()))
        unwrap()
        report("stream pool with per-stream settings vs tts_stream chunks (12 texts)", worst)
        assert worst < WAVE_ABS
        pool.close()
    finally:
        restore()


def test_stream_batch_with_kwargs_list(fast):
    """tts_stream_batch(kwargs_list=...) gives each text tts_stream's tokens with its own settings, the same chunks."""
    from test_gpu_stream_batch import _recorded_codes
    tts, cfg, clips, voices = fast
    g = torch.Generator().manual_seed(13)
    toks = [torch.randint(1, 255, (n,), generator=g).tolist() for n in torch.randint(5, 60, (6,), generator=g).tolist()]
    kl = [dict(s) for s in SETTINGS]
    kw = dict(use_deterministic_seed=3, verbose=False)          # the seed the voice latents were taken with
    restore = _one_warp_mixed()
    box, unwrap = _recorded_codes(tts, "generate_grouped_stream")
    try:
        out = list(tts.tts_stream_batch(["x"] * 6, text_tokens_list=toks, conditioning_latents_list=[voices[0]] * 6,
                                        kwargs_list=kl, **kw))
        batch_codes = box["codes"]
        unwrap()
        box1, unwrap1 = _recorded_codes(tts, "generate_stream")
        worst = 0.0
        for u in range(6):
            got = [c for v, c, _ in out if v == u]
            want = list(tts.tts_stream("x", voice_samples=clips[0], text_tokens=toks[u], **kw, **kl[u]))
            assert torch.equal(batch_codes[u], box1["codes"]), "tokens of row %d" % u
            assert [len(c) for c in got] == [len(c) for c in want], "chunks of row %d" % u
            worst = max(worst, max((a - b).abs().max().item() for a, b in zip(got, want) if a.numel()))
        unwrap1()
        report("tts_stream_batch with kwargs_list vs tts_stream chunks", worst)
        assert worst < WAVE_ABS
    finally:
        restore()


def test_tts_batch_with_kwargs_list(fast):
    """api_fast tts_batch(kwargs_list=...), some texts with typical sampling, one decoded alone (prompt of 354
    positions): entry u equals tts(texts[u], **kwargs, **kwargs_list[u]) exactly."""
    tts, cfg, clips, voices = fast
    g = torch.Generator().manual_seed(14)
    lens = torch.randint(5, 60, (8,), generator=g).tolist()
    lens[5] = 349
    toks = [torch.randint(1, 255, (n,), generator=g).tolist() for n in lens]
    kl = [dict(SETTINGS[u % len(SETTINGS)]) for u in range(8)]
    kl[2].update(typical_sampling=True, typical_mass=0.5)
    kl[5].update(typical_sampling=True)
    kl[7].update(typical_sampling=True, typical_mass=0.2)
    kw = dict(use_deterministic_seed=3, verbose=False)
    restore = _one_warp_mixed()
    try:
        got = tts.tts_batch(["x"] * 8, text_tokens_list=toks, kwargs_list=kl, **kw)
        for u in range(8):
            want = tts.tts("x", text_tokens=toks[u], **kw, **kl[u])
            assert got[u].shape == want.shape and torch.equal(got[u], want), "text %d" % u
    finally:
        restore()
