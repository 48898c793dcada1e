"""GPU: the stream pool of the api_fast path — per-row start steps in the decode step (TtbArStepArgs.row_start and the
_rows entry points), AREngine.slot_workspace, and TextToSpeech.stream_pool against tts_stream per text.

A row that joins a running batch at global step s (row_start = s - 1) must sample and capture exactly what the same
row samples and captures from step 0: the kernels are row-independent, so this holds bit for bit, in every step form.
The pool's waveforms differ from tts_stream's only through the latent source (captured vs recomputed, DESIGN §5)."""
import os

import pytest
import torch

from gpu_util import report
from test_gpu_conditioning import _clips

pytestmark = pytest.mark.gpu

WAVE_ABS = 5e-2         # stream chunks, captured vs recomputed latents (waveforms in [-1, 1])


def _mode(mode):
    from tortoise_tts_b200 import ar_engine
    E = ar_engine.AREngine
    saved = E.MODE
    E.MODE = mode

    def restore():
        E.MODE = saved
    return restore


@pytest.fixture(scope="module")
def medium():
    from tortoise_tts_b200.ar_engine import AREngine
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_autoregressive
    cfg = ModelConfig.medium()
    return cfg, AREngine(synth_autoregressive(cfg, 0, False), cfg)


@pytest.mark.parametrize("pos_mode", ["ref_kv_quirk", "train_consistent"])
@pytest.mark.parametrize("mode,C", [("fused", 4), ("mixed", 24), ("mixed", 128)])
def test_late_row_equals_the_row_from_step_zero(medium, pos_mode, mode, C):
    """Two texts (one with a prompt of 352 positions), each admitted at global step 0 into the first slots and again
    at step 37 into the last ones: the late rows' codes and captured latents equal the early rows' bit for bit. At 128
    slots the two copies run in different decode chains (two-chain mixed step, compact attention)."""
    cfg, eng = medium
    g = torch.Generator().manual_seed(3)
    toks = [torch.randint(1, 255, (n,), generator=g).tolist() + [0] for n in (30, 347)]
    voices = [torch.randn(cfg.ar_dim, generator=g).cuda() for _ in toks]
    N, late = 160, 37
    us = [torch.rand(N, generator=g).cuda() for _ in toks]
    restore = _mode(mode)
    try:
        ws = eng.slot_workspace(C, N, pos_mode=pos_mode)
        assert ws.st["mode"] == mode and len(ws.st["chains"]) == (2 if C >= 128 else 1)
        for i in range(2):
            ws.admit(i, voices[i], toks[i], us[i])
        ws.advance(late)
        for i in range(2):
            ws.admit(C - 2 + i, voices[i], toks[i], us[i])
        ws.advance(80)
        ws.check()
        codes, lat = ws.codes(), ws.latents
        n = 81
        for i in range(2):
            assert ws.tokens(i) == late + n and ws.tokens(C - 2 + i) == n
            assert torch.equal(codes[i, :n], codes[C - 2 + i, :n]), "codes of text %d" % i
            assert torch.equal(lat[i, :n], lat[C - 2 + i, :n]), "latents of text %d" % i
    finally:
        restore()


@pytest.mark.parametrize("mode", ["fused", "mixed"])
def test_zero_row_start_equals_null(medium, mode):
    """A grouped streaming decode with row_start all zeros gives the codes and latents it gives with row_start NULL."""
    cfg, eng = medium
    g = torch.Generator().manual_seed(5)
    toks = [torch.randint(1, 255, (n,), generator=g).tolist() + [0] for n in (12, 90, 40)]
    voices = [torch.randn(cfg.ar_dim, generator=g).cuda() for _ in toks]
    N = 100
    us = [torch.rand(1, N, generator=g).cuda() for _ in toks]
    restore = _mode(mode)
    try:
        runs = []
        for zero in (False, True):
            if zero:
                st = eng._dec
                for ch in st["chains"]:
                    ch["row_start"] = torch.zeros(ch["B"], dtype=torch.int32, device="cuda")
                    ch["step_handles"] = {}
                st["graph"] = None
            last = None
            for last in eng.generate_grouped_stream(voices, toks, N, 50, 50, uniforms_list=us):
                pass
            runs.append((torch.cat([c.reshape(-1) for c in last[0]]), last[2].clone()))
        assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    finally:
        eng._dec = None
        restore()


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
        tts.deterministic_state(3)
        voices.append(tts.get_conditioning_latents(c))
    bias, per_step = _raise_stop_logit(tts, cfg, voices[0].float().reshape(-1))
    report("stop logit raised by %.2f: draw probability per step" % bias, per_step)
    return tts, cfg, clips, voices


def test_pool_equals_tts_stream_per_text(fast):
    """Mixed step, one warp per stream, a pool of 8 slots: 12 texts over two voices (three with prompts of 352
    positions), each with its own seed (which also picks its conditioning crop), in three waves submitted between polls. Every stream: tts_stream's tokens bit
    for bit, its chunk count and lengths, samples within WAVE_ABS; some rows stop, some reach their cap; a slot is
    reused; no step reports a timed-out wait (checked at every observation)."""
    tts, cfg, clips, voices = fast
    g = torch.Generator().manual_seed(6)
    lens = torch.randint(5, 60, (12,), generator=g).tolist()
    lens[2] = lens[7] = lens[11] = 347
    toks = [torch.randint(1, 255, (n,), generator=g).tolist() for n in lens]
    which = [u % 2 for u in range(12)]
    restore = _one_warp_mixed()
    try:
        pool = tts.stream_pool(max_streams=8, verbose=False)
        codes, admits = {}, []
        real_finish, real_admit = pool._finish, pool.ws.admit

        def finish(s):
            codes[pool.slots[s]["sid"]] = pool.ws.codes()[s, :pool.slots[s]["tokens"]].clone()
            real_finish(s)

        def admit(slot, *a):
            admits.append(slot)
            return real_admit(slot, *a)
        pool._finish, pool.ws.admit = finish, admit
        sid_of = {}
        out = []
        for wave in ((0, 1, 2, 3, 4), (5, 6, 7, 8), (9, 10, 11)):
            for u in wave:
                sid_of[pool.submit("x", voice_samples=clips[which[u]], text_tokens=toks[u],
                                   use_deterministic_seed=3 + u)] = u
            for _ in range(3):
                out += pool.poll()
        out += list(pool.run())
        assert len(set(admits)) < len(admits), "no slot was reused: %s" % admits
        from test_gpu_stream_batch import _recorded_codes
        box, unwrap = _recorded_codes(tts, "generate_stream")
        worst, kinds = 0.0, set()
        for sid, u in sid_of.items():
            got = [(c, last) for v, c, last in out if v == sid]
            want = list(tts.tts_stream("x", voice_samples=clips[which[u]], text_tokens=toks[u],
                                       use_deterministic_seed=3 + u, verbose=False))
            assert torch.equal(codes[sid], box["codes"]), "tokens of text %d" % u
            n, cap = codes[sid].numel(), 500 - (lens[u] + 5)
            tim = pool.last_timings[sid]
            assert tim["tokens"] == n and tim["ar_ms"] > 0 and tim["prefill_ms"] > 0 and tim["hifigan_ms"] > 0
            kinds.add("cap" if n == cap else "stop")
            assert [len(c) for c, _ in got] == [len(c) for c in want], "chunks of text %d" % u
            assert [last for _, last in got] == [False] * (len(want) - 1) + [True]
            worst = max(worst, max((a - b).abs().max().item() for (a, _), b in zip(got, want) if a.numel()))
        unwrap()
        report("stream pool vs tts_stream chunks (12 texts, 8 slots, %s)" % sorted(kinds), worst)
        assert kinds == {"cap", "stop"}, "the texts should include rows that stop and rows that reach their cap"
        assert worst < WAVE_ABS
        pool.close()
    finally:
        restore()
