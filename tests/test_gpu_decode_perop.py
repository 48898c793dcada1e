"""GPU: the per-op decode step (AREngine mode "perop", one kernel per operation) at the shapes only it serves: more than
lib.AR_STEP_MAX_B = 256 candidates, or more than lib.AR_STEP_MAX_P = 352 prompt positions. tts() at its default of 512
candidates decodes here, and so does every prompt of 349 or more text tokens (counting the pad).

Kernels against float64 references: the prefix-cache layout and the step embedding bit for bit; the two partials of
ttb_ar_decode_attention (the flash kernel's split form over the prefix cache, ar_decode_attn_kernel over the candidate's
own KV) and their merge; the sampler at 512 candidates against a closed form of HF's sample(). Engine level: a row's
codes and logits do not depend on the batch it is decoded in, graph replay equals the eager loop, a 403-position prompt at
full depth against the oracle, and tts() at its default sample count. Every margin goes to the parity log (gpu_util).
"""
import math

import numpy as np
import pytest
import torch

from gpu_util import cuda_sd, rel_live, report

pytestmark = pytest.mark.gpu

V = 8194
START, STOP = 8192, 8193
NMAX = 500


def _bits(t):
    return t.contiguous().view(torch.int16)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


# ------------------------------------------------------------------ layout kernels, bit for bit
@pytest.mark.parametrize("P", [13, 353, 403])
def test_store_prefix_layout(P):
    """ar_store_prefix: the K and V columns of the prompt's qkv [P, 3D] land in the head-major caches [H, P, 64]."""
    from tortoise_tts_b200 import lib
    H = 16
    D = 64 * H
    qkv = torch.randn(P, 3 * D, generator=_gen(P), device="cuda").to(torch.bfloat16)
    pk = torch.full((H, P, 64), float("nan"), dtype=torch.bfloat16, device="cuda")
    pv = torch.full_like(pk, float("nan"))
    lib.ar_store_prefix(qkv, P, H, pk, pv)
    torch.cuda.synchronize()
    assert torch.equal(_bits(pk), _bits(qkv[:, D:2 * D].reshape(P, H, 64).transpose(0, 1)))
    assert torch.equal(_bits(pv), _bits(qkv[:, 2 * D:].reshape(P, H, 64).transpose(0, 1)))


@pytest.mark.parametrize("step", [1, NMAX - 1])
@pytest.mark.parametrize("pos_mode", [0, 1])
def test_embed_step(pos_mode, step):
    """ar_embed_step at 512 candidates: x = mel_emb[codes[:, step - 1]] + mel_pos[pos], pos = step (+ 1 in pos_mode 1)."""
    from tortoise_tts_b200 import lib
    B, D = 512, 1024
    g = _gen(7 + step + pos_mode)
    mel_emb = torch.randn(V, D, generator=g, device="cuda") * 0.05
    mel_pos = torch.randn(NMAX + 8, D, generator=g, device="cuda") * 0.05
    codes = torch.randint(0, V, (B, NMAX), generator=g, device="cuda", dtype=torch.int32)
    codes[0, step - 1], codes[B - 1, step - 1] = V - 1, 0          # first and last row of the table
    state = torch.zeros(64, dtype=torch.int32, device="cuda")
    state[0] = step
    x = torch.full((B, D), float("nan"), device="cuda")
    lib.ar_embed_step(codes, NMAX, state, mel_emb, mel_pos, B, D, pos_mode, x)
    torch.cuda.synchronize()
    pos = step + 1 if pos_mode else step
    assert torch.equal(x, mel_emb[codes[:, step - 1].long()] + mel_pos[pos])


# ------------------------------------------------------------------ decode attention: the partials and the merge
# (B, H, P, nc): across the 8-candidate CTA of ar_decode_attn_kernel, the 128-query tile of the flash kernel and the
# 64-key prefix tile with its tail (P = 13, 353, 403); nc = candidate entries incl. the new one, from the first to the
# last cache slot (Nmax = 500).
ATTN_CASES = [(512, 16, 403, 500), (512, 16, 403, 1), (512, 16, 353, 215), (512, 16, 174, 17),
              (300, 16, 403, 9), (129, 16, 353, 64), (129, 16, 13, 65),
              (1, 16, 403, 500), (1, 16, 353, 1), (257, 2, 64, 430)]
# Score offset of the dominant variants (natural-log units): the dominant side's scores are raised and the other side's
# lowered by SHIFT, so their log2-sum-exps differ by ~2 * SHIFT / ln 2 = 162 and the smaller merge weight exp2 underflows
# to exactly 0 in fp32 (below 2^-149).
SHIFT = 56.0


def _attn_inputs(B, H, P, variant, seed):
    D = 64 * H
    g = _gen(seed)

    def rn(*s):
        return torch.randn(*s, generator=g, device="cuda")
    qkv, pk, pv = rn(B, 3 * D), rn(H, P, 64), rn(H, P, 64)
    ck, cv = rn(B, H, NMAX, 64), rn(B, H, NMAX, 64)
    if variant == "rising":
        # the running max of the prefix scores grows by far more than 2^8 across tiles: the flash kernel's lazy rescale
        pk *= (1 + torch.arange(P, device="cuda") / 32).view(1, P, 1)
    elif variant in ("prefix_dominant", "own_dominant"):
        qkv[:, :D].view(B, H, 64)[..., 0] = 8.0                       # q . k gets 8 k_0: a score of 0.125 * 8 * k_0
        sp, so = (SHIFT, -SHIFT) if variant == "prefix_dominant" else (-SHIFT, SHIFT)
        pk[..., 0] = sp
        ck[..., 0] = so
        qkv[:, D:2 * D].view(B, H, 64)[..., 0] = so                   # the new key is one of the candidate's own
    return [t.to(torch.bfloat16) for t in (qkv, pk, pv, ck, cv)]


@pytest.mark.parametrize("variant", ["plain", "rising", "prefix_dominant", "own_dominant"])
@pytest.mark.parametrize("B,H,P,nc", ATTN_CASES)
def test_decode_attention_partials_and_merge(B, H, P, nc, variant):
    """ttb_ar_decode_attention at step nc: the KV append, each partial (normalised fp32 row + log2-sum-exp) against
    float64, and the merged bf16 row over [prefix | own keys].

    Bounds. Candidate partial (ar_decode_attn_kernel): fp32 throughout, o within 5e-5 of its scale, LSE within 1e-4
    (log2 units; fp32 rounding of scores up to ~80 in the dominant variants). Prefix partial (flash kernel): the softmax
    weights are rounded to bf16 for the P V product (2^-9 relative each), o within 8e-3 of its scale as the mma bound of
    test_gpu_ar_step; its row sum and LSE come from the unrounded fp32 weights, so the LSE has the candidate side's
    bound, 1e-4. Merged row: within 6e-3, as test_step_attention_phase. Largest measured (H100 80GB HBM3, 700 W): o 7.8e-6
    / LSE 2.8e-5 candidate side, o 2.9e-3 / LSE 1.9e-5 prefix side, merged 5.2e-3."""
    from tortoise_tts_b200 import lib
    D = 64 * H
    qkv, pk, pv, ck, cv = _attn_inputs(B, H, P, variant, seed=B * 1000 + P + nc)
    slot = nc - 1
    want_ck, want_cv = ck.clone(), cv.clone()
    want_ck[:, :, slot] = qkv[:, D:2 * D].reshape(B, H, 64)
    want_cv[:, :, slot] = qkv[:, 2 * D:].reshape(B, H, 64)
    state = torch.zeros(64, dtype=torch.int32, device="cuda")
    state[0] = nc
    out = torch.full((B, D), float("nan"), dtype=torch.bfloat16, device="cuda")
    so = torch.full((2, B, D), float("nan"), device="cuda")
    slse = torch.full((2, B, H), float("nan"), device="cuda")
    lib.ar_decode_attention(qkv, pk, pv, ck, cv, state, B, H, P, NMAX, out, so, slse)
    torch.cuda.synchronize()
    assert torch.equal(_bits(ck), _bits(want_ck)), "K cache: the new row is not the qkv K column, or another row changed"
    assert torch.equal(_bits(cv), _bits(want_cv)), "V cache: the new row is not the qkv V column, or another row changed"
    del want_ck, want_cv
    # float64 reference, in chunks of candidates (peak memory: two [64, H, nc, 64] float64 blocks)
    err = dict(o_own=0.0, lse_own=0.0, o_prefix=0.0, lse_prefix=0.0, out=0.0)
    scale = dict(o_own=0.0, o_prefix=0.0, out=0.0)
    pk64, pv64 = pk.double(), pv.double()
    for b0 in range(0, B, 64):
        b1 = min(B, b0 + 64)
        q = qkv[b0:b1, :D].double().view(-1, H, 64)
        s_p = torch.einsum("bhd,hpd->bhp", q, pk64) * 0.125
        kc, vc = ck[b0:b1, :, :nc].double(), cv[b0:b1, :, :nc].double()     # = the old rows + the new one (checked above)
        s_c = torch.einsum("bhd,bhnd->bhn", q, kc) * 0.125
        lse_p, lse_c = torch.logsumexp(s_p, -1), torch.logsumexp(s_c, -1)
        o_p = torch.einsum("bhp,hpd->bhd", torch.softmax(s_p, -1), pv64)
        o_c = torch.einsum("bhn,bhnd->bhd", torch.softmax(s_c, -1), vc)
        lse = torch.logaddexp(lse_p, lse_c)
        o = o_p * torch.exp(lse_p - lse).unsqueeze(-1) + o_c * torch.exp(lse_c - lse).unsqueeze(-1)
        for key, got, want in (("o_prefix", so[0, b0:b1], o_p), ("o_own", so[1, b0:b1], o_c), ("out", out[b0:b1], o)):
            err[key] = max(err[key], (got.double().view(-1, H, 64) - want).abs().max().item())
            scale[key] = max(scale[key], want.abs().max().item())
        err["lse_prefix"] = max(err["lse_prefix"], (slse[0, b0:b1].double() - lse_p / math.log(2)).abs().max().item())
        err["lse_own"] = max(err["lse_own"], (slse[1, b0:b1].double() - lse_c / math.log(2)).abs().max().item())
    r = {k: (err[k] / max(scale[k], 1e-6) if k in scale else err[k]) for k in err}
    for k, v in r.items():
        report("perop decode attention %s B=%d H=%d P=%d nc=%d %s" % (k, B, H, P, nc, variant), v)
    assert r["o_own"] < 5e-5 and r["lse_own"] < 1e-4, r
    assert r["o_prefix"] < 8e-3 and r["lse_prefix"] < 1e-4, r
    assert r["out"] < 6e-3, r


# ------------------------------------------------------------------ sampler at 512 candidates
def _hf_sample(row, seen, u, temperature, top_k, top_p, rep):
    """One HF sample() step in float64 closed form: repetition penalty over `seen`, temperature, top-k keeping every tie
    of the k-th score, top-p on the exclusive prefix mass in descending order (ties by ascending id, as the kernel orders
    them), inverse-CDF draw of `u` over the kept set. Returns (token, widened kept set, boundary flag).

    A row is a boundary row when fp32 rounding can decide it: u within 1e-5 of a CDF step, an exclusive prefix mass within
    1e-5 of top_p, or a DISTINCT score within 1e-6 relative of the k-th one. Exact ties are not boundaries: tied tokens
    have bit-identical processed scores in the kernel too, and HF keeps every one of them. The widened set adds what
    such a rounding could also keep."""
    s = row.astype(np.float64)
    idx = np.fromiter(seen, dtype=np.int64)
    v = s[idx]
    s[idx] = np.where(v < 0, v * rep, v / rep)
    s = s / temperature
    order = np.lexsort((np.arange(s.size), -s))            # descending score, ascending id
    ss = s[order]
    kth = ss[top_k - 1]
    n_ge = int(np.searchsorted(-ss, -kth, side="right"))    # every score >= the k-th
    near = np.abs(ss - kth) <= 1e-6 * abs(kth)
    near_tie = bool(near[n_ge:].any())
    p = np.exp(ss[:n_ge] - ss[0])
    p /= p.sum()
    excl = np.cumsum(p) - p
    keep = excl < top_p
    keep[0] = True
    nk = int(keep.sum())                                    # a prefix: excl increases
    kp = p[:nk] / p[:nk].sum()
    cdf = np.cumsum(kp)
    j = min(int(np.searchsorted(cdf, u, side="right")), nk - 1)
    boundary = near_tie or bool((np.abs(excl[1:] - top_p) < 1e-5).any()) or bool((np.abs(cdf - u) < 1e-5).any())
    wide = set(order[:n_ge][(excl < top_p + 1e-5) | (np.arange(n_ge) == 0)].tolist())
    wide |= set(order[n_ge:][near[n_ge:]].tolist())
    return int(order[j]), wide, boundary


def _seen_mask(seen):
    m = np.zeros((len(seen), (V + 31) // 32), dtype=np.uint32)
    for b, ids in enumerate(seen):
        for t in ids:
            m[b, t >> 5] |= np.uint32(1 << (t & 31))
    return torch.from_numpy(m.view(np.int32))


SAMPLING = {"tts_defaults": (0.8, 50, 0.8, 2.0), "greedy": (1.0, 1, 1.0, 1.0), "sharp": (0.3, 50, 0.95, 4.0)}


@pytest.mark.parametrize("params", list(SAMPLING))
def test_sampler_512(params):
    """ar_sample at 512 candidates, three launches as generate() runs them (the prefill row broadcast with ld_logits = 0,
    then one row per candidate), the kernel's own draws fed back through `seen`; then one launch with every row finished.
    Rows: logit scales 0.5 .. 6, entries pinned at -1e4, three tokens tied at the 50th score (row 40), the whole top 50
    tied (row 41), one row that draws the stop token (row 77 at the second launch), rows 5, 300, 511 finished."""
    from tortoise_tts_b200 import lib
    temperature, top_k, top_p, rep = SAMPLING[params]
    B, NC = 512, 5
    FIN, TIE3, TIE50, STOPROW = (5, 300, 511), 40, 41, 77
    rng = np.random.default_rng(sorted(SAMPLING).index(params) + 11)
    u = torch.from_numpy(rng.random((B, 3), dtype=np.float32))
    scales = np.linspace(0.5, 6.0, B, dtype=np.float32)[:, None]
    seen_ids = [{1, START} for _ in range(B)]
    seen = _seen_mask(seen_ids).cuda()
    codes = torch.full((B, NC), -1, dtype=torch.int32, device="cuda")
    finished = torch.zeros(B, dtype=torch.int32, device="cuda")
    finished[list(FIN)] = 1
    state = torch.zeros(64, dtype=torch.int32, device="cuda")
    u_dev = u.cuda()

    def pinned(rows):
        rows[:, STOP] = -1e4
        for r in rows:
            r[rng.integers(0, V, 8)] = -1e4
        return rows
    checked = nb = 0
    for launch in range(3):
        if launch == 0:
            logits = pinned(rng.standard_normal((1, V), dtype=np.float32) * 2.0)
        else:
            logits = pinned(rng.standard_normal((B, V), dtype=np.float32) * scales)
            for r, ntie in ((TIE3, 3), (TIE50, 50)):
                row = logits[r]
                row[list(seen_ids[r])] = -50.0                # no tied token is penalised: the ties hold after it
                o = np.argsort(-row, kind="stable")
                if ntie == 3:
                    row[o[60]] = row[o[61]] = row[o[49]]
                else:
                    row[o[:50]] = row[o[0]]
            if launch == 1:
                logits[STOPROW, STOP] = 60.0
        fin_before = finished.cpu().bool()
        codes_before = codes.cpu()
        lib.ar_sample(torch.from_numpy(logits).cuda(), 0 if launch == 0 else V, V, B, u_dev, 3, seen, codes, NC, finished,
                      state, temperature, top_k, top_p, rep, STOP, advance=True)
        torch.cuda.synchronize()
        st, c = state.cpu(), codes.cpu()
        assert int(st[0]) == launch + 1 and int(st[3]) == 0, st[:4]
        other = torch.arange(NC) != launch
        assert torch.equal(c[:, other], codes_before[:, other]), "codes written outside column %d" % launch
        drawn = c[:, launch]
        assert (drawn[fin_before] == STOP).all()
        mism = []
        for b in range(B):
            if fin_before[b]:
                continue
            tok = int(drawn[b])
            want, wide, boundary = _hf_sample(logits[0 if launch == 0 else b], seen_ids[b], float(u[b, launch]),
                                              temperature, top_k, top_p, rep)
            checked += 1
            nb += int(boundary)
            assert tok in wide, (launch, b, tok, want)
            if not boundary and tok != want:
                mism.append((b, tok, want))
            seen_ids[b].add(tok)
        assert not mism, "launch %d: tokens differ from the closed form on non-boundary rows %s" % (launch, mism[:8])
        fin_now = fin_before | (drawn == STOP)
        if launch == 1:
            assert bool(fin_now[STOPROW])
        assert torch.equal(finished.cpu().bool(), fin_now)
        assert int(st[1]) == int(bool(fin_now.all())) == 0
        assert torch.equal(seen.cpu(), _seen_mask(seen_ids)), "seen bitmask is not {1, start} + the draws"
    report("perop sampler 512 %s boundary-row fraction" % params, nb / checked)
    assert nb < 0.02 * checked, (nb, checked)
    # every row finished: stop tokens only, the all-finished flag set, the step still advanced
    finished.fill_(1)
    lib.ar_sample(torch.zeros(B, V, device="cuda"), V, V, B, u_dev, 3, seen, codes, NC, finished, state, temperature, top_k,
                  top_p, rep, STOP, advance=True)
    torch.cuda.synchronize()
    st = state.cpu()
    assert int(st[0]) == 4 and int(st[1]) == 1 and int(st[3]) == 0, st[:4]
    assert (codes[:, 3].cpu() == STOP).all() and (codes[:, 4].cpu() == -1).all()


# ------------------------------------------------------------------ engine level
ROWS = [0, 7, 8, 127, 128, 255, 256, 257, 510, 511]


def _text(n, seed):
    """n text tokens, the last one the pad: prompt P = n + 4."""
    return torch.randint(1, 255, (n - 1,), generator=torch.Generator().manual_seed(seed)).tolist() + [0]


@pytest.fixture(scope="module")
def medium_ar():
    """Full width, 2 layers; the stop token is suppressed, so every row decodes every step."""
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_autoregressive
    cfg = ModelConfig.medium()
    return cfg, synth_autoregressive(cfg, 1, True)          # = synth_all(cfg, 1, suppress_stop=True)["autoregressive"]


@pytest.mark.parametrize("P", [403, 174])
def test_rows_do_not_depend_on_the_batch(medium_ar, monkeypatch, P):
    """The same 10 rows decoded inside a batch of 512 and as a batch of 10: codes and the logits the sampler sees must be
    BIT-identical. Every kernel of the per-op step is row-independent; the mel_head GEMM takes the 128x256 kernel at 512
    rows and the one-tile kernel at 10, which test_gpu_gemm_ws holds bit-identical to each other."""
    from tortoise_tts_b200 import lib
    from tortoise_tts_b200.ar_engine import AREngine
    cfg, sd = medium_ar
    N = 16
    text = _text(P - 4, P)
    g = torch.Generator().manual_seed(P + 1)
    cond = torch.randn(1, cfg.ar_dim, generator=g)
    u = torch.rand(512, N, generator=g)
    eng = AREngine(sd, cfg)
    tr_all = []
    codes_all = eng.generate(cond, text, 512, N, uniforms=u, trace_logits=tr_all)
    assert eng._dec["mode"] == "perop" and eng._dec["P"] == P
    if P <= lib.AR_STEP_MAX_P:
        monkeypatch.setattr(AREngine, "MODE", "perop")      # 10 rows at this prompt would take the one-kernel step
    tr = []
    codes = eng.generate(cond, text, len(ROWS), N, uniforms=u[ROWS], trace_logits=tr)
    assert eng._dec["mode"] == "perop" and eng._dec["B"] == len(ROWS)
    rows = torch.tensor(ROWS, device=codes.device)
    diff = max((tr[n] - tr_all[n][rows]).abs().max().item() for n in range(N))
    report("perop rows vs batch P=%d: max |logit difference|" % P, diff)
    assert torch.equal(codes, codes_all[rows])
    assert all(torch.equal(tr[n], tr_all[n][rows]) for n in range(N))


def test_graph_replay_equals_eager_512(medium_ar):
    """generate()'s default: the per-op step captured as a CUDA graph (the decode attention forks onto the library's side
    stream and joins back inside it), replayed in blocks of 4 steps; twice, against the eager loop, at B = 512, P = 403."""
    from tortoise_tts_b200.ar_engine import AREngine
    cfg, sd = medium_ar
    B, N = 512, 16
    text = _text(399, 5)
    g = torch.Generator().manual_seed(6)
    cond = torch.randn(1, cfg.ar_dim, generator=g)
    u = torch.rand(B, N, generator=g)
    eng = AREngine(sd, cfg)
    eager = eng.generate(cond, text, B, N, uniforms=u, use_graph=False)
    assert eng._dec["mode"] == "perop" and eng._dec["graph"] is None
    for _ in range(2):
        got = eng.generate(cond, text, B, N, uniforms=u, use_graph=True, stop_check_every=4)
        assert eng._dec["graph"] is not None
        assert torch.equal(got, eager), "CUDA-graph replay of the per-op step differs from the eager loop"


def test_long_prompt_full_depth_vs_oracle():
    """30 layers, full width, 399 text tokens (P = 403): the logits the sampler sees at 48 consecutive steps against the
    oracle's teacher-forced logits of the produced sequence (fp32, on the GPU), and every token inside the kept set of
    the oracle's sample_step on those logits. The analogue of test_gpu_parity_prod's prompt-174 test."""
    from tortoise_tts_b200.ar_engine import AREngine
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_autoregressive
    from oracle import ar
    cfg = ModelConfig.full()
    sd = synth_autoregressive(cfg, 0, True)
    text = _text(399, 2)
    g = torch.Generator().manual_seed(3)
    cond = torch.randn(1, cfg.ar_dim, generator=g) * 0.5
    B, N = 4, 48
    u = torch.rand(B, N, generator=g)
    eng = AREngine(sd, cfg)
    tr = []
    codes = eng.generate(cond, text, B, N, uniforms=u, trace_logits=tr).long()
    assert eng._dec["mode"] == "perop" and eng._dec["P"] == 403
    seen = torch.stack(tr, 1)
    with torch.no_grad(), torch.device("cuda"):
        want = ar.teacher_forced_logits(cuda_sd(sd), cfg, cond.cuda(), text, codes[:, :-1].cuda())
    r = rel_live(seen, want.to(seen.device))
    report("perop AR decode-loop logits P=403 L=30 (48 steps, live-logit scale)", r)
    assert r < 0.03
    seen, codes = seen.cpu(), codes.cpu()
    for b in range(B):
        prev = {1, cfg.start_mel_token}
        for n in range(N):
            tok = int(codes[b, n])
            _, kept, _ = ar.sample_step(seen[b, n], prev, float(u[b, n]))
            assert tok in set(kept.tolist()), (b, n, tok)
            prev.add(tok)


def test_tts_default_sample_count():
    """tts() with num_autoregressive_samples at its default (512): the decode runs per-op as a captured graph, the
    waveform is finite, and a second call with the same seed reuses the graph and returns the same waveform."""
    from tortoise_tts_b200.api import TextToSpeech
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_all
    cfg = ModelConfig.small()
    tts = TextToSpeech(state_dicts=synth_all(cfg, seed=0, suppress_stop=False), config=cfg, enable_redaction=False)
    cl = (torch.randn(1, cfg.ar_dim, generator=torch.Generator().manual_seed(2)),
          torch.randn(1, 2 * cfg.diff_dim, generator=torch.Generator().manual_seed(3)) * 0.3)
    kw = dict(text_tokens=[12, 40, 7, 99, 3], conditioning_latents=cl, use_deterministic_seed=5, max_mel_tokens=16,
              diffusion_iterations=4, verbose=False)
    wav = tts.tts("x", **kw)
    dec = tts.autoregressive._dec
    assert dec["mode"] == "perop" and dec["B"] == 512 and dec["graph"] is not None
    graph = dec["graph"]
    assert wav.numel() > 0 and torch.isfinite(wav).all()
    wav2 = tts.tts("x", **kw)
    assert tts.autoregressive._dec["graph"] is graph
    assert torch.equal(wav2, wav)
