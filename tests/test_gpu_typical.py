"""GPU: the typical-set filter of the fused sampler (ttb_ar_sample_typical, csrc/ar.cu) against the oracle
(tests/typical_oracle.py, pinned to the reference's TypicalLogitsWarper by tests/test_typical_vs_reference.py), and
through the AR engine and the facade."""
import pytest
import torch

import typical_oracle

pytestmark = pytest.mark.gpu

V = 8194
TOL = 1e-5


def _penalised(row, prev, rep=2.0):
    s = row.clone().float()
    idx = torch.tensor(sorted(set(int(i) for i in prev)), dtype=torch.long)
    v = s[idx]
    s[idx] = torch.where(v < 0, v * rep, v / rep)
    return s


def _oracle(row, prev, u, mass, **kw):
    """(token, kept ids, T widened by the next key group when the row sits at a boundary, boundary flag)."""
    tok, kept, _ = typical_oracle.sample_step(row, prev, u, typical_mass=mass, **kw)
    s = _penalised(row, prev)
    keep, v = typical_oracle.typical_keep(s, mass)
    lp = torch.log_softmax(s.double(), -1)
    key = (-lp - (-(lp * lp.exp()).nansum())).abs()
    p = lp.exp()
    kf = key.float()
    below = p[kf < v].sum().item()
    upto = p[kf <= v].sum().item()
    above = kf[kf > v]
    vn = above.min().item() if above.numel() else v
    boundary = abs(below - mass) < TOL or abs(upto - mass) < TOL or (vn - v) <= TOL * max(v, 1e-6) or \
        ((kf - v).abs() <= TOL * max(v, 1e-6)).sum().item() > (kf == v).sum().item()
    wide = keep | (kf <= vn * (1 + TOL) + TOL) if boundary else keep
    return tok, kept.tolist(), wide, boundary


def _launch(lib, logits, ld, u, seen, mass, B, top_k=50, top_p=0.8, fin=None):
    N = u.shape[1]
    codes = torch.full((B, N), -1, dtype=torch.int32, device="cuda")
    fin = torch.zeros(B, dtype=torch.int32, device="cuda") if fin is None else fin.clone()
    state = torch.zeros(64, dtype=torch.int32, device="cuda")
    lib.ar_sample_typical(logits, ld, V, B, u, N, seen.clone(), codes, N, fin, state, 0.8, top_k, top_p, 2.0, 8193,
                          mass, advance=True)
    torch.cuda.synchronize()
    return codes[:, 0].cpu(), state


def _seen(prev):
    seen = torch.zeros(len(prev), (V + 31) // 32, dtype=torch.int32)
    for b, ids in enumerate(prev):
        for t in set(ids):
            seen[b, t // 32] |= (1 << (t % 32)) if t % 32 < 31 else -(1 << 31)
    return seen.cuda()


@pytest.mark.parametrize("mass", [0.2, 0.5, 0.9, 0.999])
def test_kernel_matches_oracle(mass):
    from tortoise_tts_b200 import lib
    g = torch.Generator().manual_seed(int(mass * 1000))
    B = 256
    logits = torch.randn(B, V, generator=g) * torch.linspace(0.5, 6.0, B).unsqueeze(1)
    u = torch.rand(B, 2, generator=g)
    prev = [[1, 8192] + torch.randint(0, 8192, (20,), generator=g).tolist() for _ in range(B)]
    fin = torch.zeros(B, dtype=torch.int32, device="cuda")
    fin[7] = 1
    codes, state = _launch(lib, logits.cuda(), V, u.cuda(), _seen(prev), mass, B, fin=fin)
    assert int(state[0]) == 1 and int(state[1]) == 0
    mism = nb = 0
    for b in range(B):
        if b == 7:
            assert int(codes[b]) == 8193
            continue
        tok, kept, wide, boundary = _oracle(logits[b], prev[b], float(u[b, 0]), mass)
        nb += int(boundary)
        assert bool(wide[int(codes[b])])                  # never outside T (widened only at a boundary)
        if tok != int(codes[b]):
            mism += 1
            assert boundary or int(codes[b]) in kept      # a top-p / inverse-CDF rounding boundary otherwise
    assert mism <= 3, (mism, nb)


def _adversarial():
    g = torch.Generator().manual_seed(21)
    rows = []
    peaked = torch.randn(V, generator=g) * 0.1
    peaked[:5] = torch.tensor([20.0, 19.8, 19.6, 19.4, 19.2])       # |T| = 5 < top_k
    rows.append(peaked)
    single = torch.randn(V, generator=g)
    single[777] = 40.0                                               # |T| = 1
    rows.append(single)
    for levels in ([2.0, 0.0], [1.0, 0.5, -3.0], [0.0], [4.0, 1.0, 0.0, -1.0]):   # every key tied with a whole level
        rows.append(torch.tensor(levels)[torch.randint(0, len(levels), (V,), generator=g)])
    for scale in (0.3, 3.0, 12.0):
        rows.append(torch.randn(V, generator=g) * scale)
    few = torch.full((V,), -30.0)
    few[torch.randint(0, V, (60,), generator=g)] = torch.randn(60, generator=g) * 2      # mass on 60 tokens
    rows.append(few)
    return torch.stack(rows)


@pytest.mark.parametrize("mass", [0.05, 0.2, 0.5, 0.9, 0.999, 1.0])
@pytest.mark.parametrize("top_p", [0.8, 1.0])
def test_never_outside_the_typical_set(mass, top_p):
    """Hard check over adversarial rows, with uniforms that include the draw of the last kept token (u just below 1)."""
    from tortoise_tts_b200 import lib
    rows = _adversarial()
    us = torch.tensor([0.0, 0.5, 0.999, 1.0 - 2.0 ** -24])
    R = rows.shape[0]
    logits = rows.repeat_interleave(len(us), 0)
    u = us.repeat(R).unsqueeze(1)
    prev = [[1, 8192]] * (R * len(us))
    codes, _ = _launch(lib, logits.cuda(), V, u.cuda(), _seen(prev), mass, R * len(us), top_p=top_p)
    for r in range(R):
        _, _, wide, _ = _oracle(rows[r], [1, 8192], 0.5, mass, top_p=top_p)
        for j in range(len(us)):
            assert bool(wide[int(codes[r * len(us) + j])]), (r, j)


def test_distribution():
    """chi-square of 4000 draws from one row against the oracle's kept probabilities."""
    from tortoise_tts_b200 import lib
    g = torch.Generator().manual_seed(6)
    B, mass = 4000, 0.5
    row = torch.randn(1, V, generator=g) * 3
    u = torch.rand(B, 1, generator=g)
    codes, _ = _launch(lib, row.cuda(), 0, u.cuda(), _seen([[]] * B), mass, B)
    _, kept, kp = typical_oracle.sample_step(row[0], [], 0.5, typical_mass=mass)
    counts = torch.bincount(codes.long(), minlength=V)[kept]
    assert counts.sum().item() == B
    exp = kp * B
    chi2 = ((counts - exp) ** 2 / exp).sum().item()
    assert chi2 < 3 * len(kp) + 20, chi2


def test_deterministic():
    from tortoise_tts_b200 import lib
    g = torch.Generator().manual_seed(7)
    B = 256
    logits = (torch.randn(B, V, generator=g) * 3).cuda()
    u = torch.rand(B, 1, generator=g).cuda()
    seen = _seen([[1, 8192]] * B)
    a, _ = _launch(lib, logits, V, u, seen, 0.7, B)
    b, _ = _launch(lib, logits, V, u, seen, 0.7, B)
    assert torch.equal(a, b)


def test_mass_out_of_range_is_an_error():
    from tortoise_tts_b200 import lib
    u = torch.rand(1, 1).cuda()
    with pytest.raises(lib.TtbError):
        _launch(lib, torch.randn(1, V).cuda(), V, u, _seen([[]]), 0.0, 1)


TEXT = [12, 40, 7, 99, 3]


def test_engine_modes_and_oracle(monkeypatch):
    """AREngine.generate with the filter on: one- and two-chain decodes agree bit for bit, CUDA-graph replay equals the
    eager loop in every mode, every token is the oracle's draw (or, at a boundary of T, in the widened set) on the
    logits the sampler saw, and a change of the mass captures a new graph."""
    from tortoise_tts_b200.ar_engine import AREngine
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_all
    cfg = ModelConfig.small()
    sd = synth_all(cfg, seed=0, suppress_stop=False)["autoregressive"]
    B, N, mass = 8, 10, 0.6
    u = torch.rand(B, N, generator=torch.Generator().manual_seed(8))
    cond = torch.randn(cfg.ar_dim, generator=torch.Generator().manual_seed(9))
    monkeypatch.setattr(AREngine, "CHAINS_MIN_B", 2)
    outs = {}
    for mode, chains in (("fused", 1), ("mixed", 1), ("mixed", 2)):
        monkeypatch.setattr(AREngine, "MODE", mode)
        monkeypatch.setattr(AREngine, "CHAINS", chains)
        eng = AREngine(sd, cfg)
        outs[(mode, chains)] = eng.generate(cond, TEXT, B, N, uniforms=u, typical_mass=mass).cpu()
        assert eng._dec["mode"] == mode and len(eng._dec["chains"]) == chains
        eager = eng.generate(cond, TEXT, B, N, uniforms=u, typical_mass=mass, use_graph=False).cpu()
        assert torch.equal(eager, outs[(mode, chains)])
    # one and two chains run the same kernels per row: bit for bit. (The one-kernel fused step rounds its GEMMs at other
    # points than the per-op step, so fused against mixed agrees to bf16 noise only, with or without the filter.)
    first = outs[("mixed", 1)]
    assert torch.equal(outs[("mixed", 2)], first)
    # graph cache keyed on the mass
    g0 = eng._dec["graph"]
    eng.generate(cond, TEXT, B, N, uniforms=u, typical_mass=mass)
    assert eng._dec["graph"] is g0
    eng.generate(cond, TEXT, B, N, uniforms=u, typical_mass=0.3)
    assert eng._dec["graph"] is not g0 and eng._dec["graph_params"]["typical_mass"] == pytest.approx(0.3)
    # every token against the oracle on the logits the sampler saw (eager run with the logits trace)
    monkeypatch.setattr(AREngine, "MODE", "mixed")
    monkeypatch.setattr(AREngine, "CHAINS", 1)
    eng = AREngine(sd, cfg)
    tr = []
    codes = eng.generate(cond, TEXT, B, N, uniforms=u, typical_mass=mass, trace_logits=tr).cpu().long()
    assert torch.equal(codes, first)
    mism = 0
    for b in range(B):
        seen = {1, cfg.start_mel_token}
        for n in range(N):
            if n > 0 and int(codes[b, n - 1]) == cfg.stop_mel_token:
                assert int(codes[b, n]) == cfg.stop_mel_token
                continue
            tok, kept, wide, boundary = _oracle(tr[n][b].cpu(), seen, float(u[b, n]), mass)
            assert bool(wide[int(codes[b, n])]), (b, n)
            if tok != int(codes[b, n]):
                mism += 1
                assert boundary or int(codes[b, n]) in kept
            seen.add(int(codes[b, n]))
    assert mism <= 3, mism


def test_tts_end_to_end():
    from tortoise_tts_b200.api import TextToSpeech
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_all
    cfg = ModelConfig.small()
    tts = TextToSpeech(state_dicts=synth_all(cfg, seed=0, suppress_stop=False), config=cfg, kv_cache=True,
                       enable_redaction=False)
    cl = (torch.randn(1, cfg.ar_dim, generator=torch.Generator().manual_seed(2)),
          torch.randn(1, 2 * cfg.diff_dim, generator=torch.Generator().manual_seed(3)) * 0.3)
    kw = dict(text_tokens=TEXT, conditioning_latents=cl, use_deterministic_seed=5, max_mel_tokens=24,
              num_autoregressive_samples=8, diffusion_iterations=4, verbose=False, cond_free=False)
    wav = tts.tts("x", typical_sampling=True, typical_mass=0.8, **kw)
    assert torch.isfinite(wav).all() and wav.numel() > 0
