"""CPU: the DDIM sampler option (DiffusionEngine.sample(sampler="ddim"), tts(diffusion_sampler="ddim")) without a GPU.

A torch emulation of ttb_ddim_step (csrc/misc.cu ddim_step_kernel), defined here, against one update of the DDIM oracle
(tests/ddim_oracle.py); the oracle loop against the reference's ddim_sample_loop outputs in tests/golden/ddim_small_v1.pt;
the engine's host orchestration on the emulated kernel library against the same fixture; the facade's argument checks."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import ddim_oracle
import lib_emu
from tortoise_tts_b200.config import ModelConfig
from tortoise_tts_b200.diffusion_engine import make_ddim_schedule
from tortoise_tts_b200.synth import synth_all

GOLD = os.path.join(os.path.dirname(__file__), "golden", "ddim_small_v1.pt")


def ddim_step(model_out, out_bstride, ld_out, x, x_bf16, ld_xb, noise, tables, step, S, Cc, iters, cond_free,
              cond_free_k, mel_out=None, parity_stride=0):
    """torch emulation of lib.ddim_step (same signature): fp32 element-wise arithmetic in the kernel's order."""
    assert parity_stride == 0, "the peer-exchange area exists on GPUs only"
    call = int(step[0])
    i = iters - 1 - call
    tb = lib_emu._v(tables, (5, iters), (iters, 1))
    mo = lib_emu._v(model_out, (2 if cond_free else 1, S, Cc), (out_bstride, ld_out, 1))
    eps = mo[0]
    if cond_free:
        cfk = cond_free_k * (1 - i / iters)
        eps = torch.tensor(1 + cfk, dtype=torch.float32) * eps - torch.tensor(cfk, dtype=torch.float32) * mo[1]
    xx = lib_emu._v(x, (S, Cc), (Cc, 1))
    sx = tb[0, i] * xx
    x0 = (sx - tb[1, i] * eps).clamp(-1, 1)
    e2 = (sx - x0) / tb[1, i]
    nv = 0.0 if noise is None else lib_emu._v(noise, (iters, S, Cc), (S * Cc, Cc, 1))[call]
    xn = (tb[2, i] * x0 + tb[3, i] * e2) + (0.0 if i == 0 else 1.0) * tb[4, i] * nv
    xx.copy_(xn)
    if x_bf16 is not None:
        lib_emu._v(x_bf16, (S, Cc), (ld_xb, 1)).copy_(xn.to(torch.bfloat16))
    if mel_out is not None and i == 0:
        lib_emu._v(mel_out, (Cc, S), (S, 1)).copy_((((xn + 1) / 2) * (2.3143386840820312 + 11.512925148010254)
                                                    - 11.512925148010254).t())


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD)


@pytest.mark.parametrize("eta", [0.0, 0.7, 1.0])
@pytest.mark.parametrize("cond_free", [True, False])
def test_kernel_emulation_matches_oracle_step(eta, cond_free):
    """The kernel's arithmetic on make_ddim_schedule's tables == ddim_update on fp32 tables computed as the reference
    computes them, at the first, a middle and the last call of a 30-step chain."""
    iters, S, Cc = 30, 37, 100
    _, tables = make_ddim_schedule(iters, eta)
    tb_o, _ = ddim_oracle.ddim_tables(iters)
    g = torch.Generator().manual_seed(3)
    x_init = torch.randn(S, Cc, generator=g) * 3
    mo = torch.randn(2, S, 2 * Cc, generator=g)
    noise = torch.randn(iters, S, Cc, generator=g)
    for call in (0, 14, iters - 1):
        i = iters - 1 - call
        x = x_init.clone()
        mel = torch.zeros(Cc, S)
        ddim_step(mo, S * 2 * Cc, 2 * Cc, x, None, 0, noise, torch.from_numpy(tables), torch.tensor([call]), S, Cc,
                  iters, cond_free, 2.0, mel)
        want = ddim_oracle.ddim_update(tb_o, i, iters, x_init, mo[0, :, :Cc], mo[1, :, :Cc] if cond_free else None,
                                       noise[call], eta, 2.0)
        err = (x - want).abs().max().item() / max(want.abs().max().item(), 1.0)
        assert err < 1e-5, (call, err)
        if i == 0:
            # the last step returns the clamped x0: the mel lies inside the denormalised range
            assert x.abs().max().item() <= 1.0
            assert -11.5131 <= mel.min().item() and mel.max().item() <= 2.3144


def test_oracle_matches_golden(gold):
    """tests/ddim_oracle.py == the reference's ddim_sample_loop (same torch RNG draws) on the small checkpoint."""
    cfg = ModelConfig.small()
    sd = synth_all(cfg, seed=0, suppress_stop=False)["diffusion"]
    assert abs(float(sum(v.double().sum() for v in sd.values())) - gold["weights_checksum"]) < 1e-6 * max(
        1.0, abs(gold["weights_checksum"]))
    with torch.no_grad():
        for case in gold["cases"]:
            n = case["iters"]
            x = ddim_oracle.ddim_sample_loop(sd, cfg, gold["code_emb"], gold["noise0"], gold["step_noise"][:n], n,
                                             case["eta"], case["cond_free"], gold["cond_free_k"])
            err = (x - case["x0"]).abs().max().item()
            assert err < 1e-3, (case["iters"], case["eta"], case["cond_free"], err)


@pytest.fixture()
def emu():
    import tortoise_tts_b200.lib as real
    saved = lib_emu.install()
    saved.setdefault("ddim_step", real.ddim_step)
    real.ddim_step = ddim_step
    yield
    lib_emu.uninstall(saved)


def check_ddim_mel(mel, ref, what):
    """Bound on a DDIM mel of the small synthetic checkpoint against the reference's loop with the same noise.

    The emulation is the fp32 oracle with bf16-rounded GEMM operands. On the fixture's short chains its drift from the
    reference is 2-4x that of the p sampler (measured max / p99.9 / rms of |mel difference|, range 13.8: 6.55 / 1.73 /
    0.16 at 6 steps, eta 0, CFG; 8.99 / 4.19 / 0.27 at 4 steps, eta 0, no CFG; 0.98 / 0.58 / 0.08 at eta 1). Perturbing
    only the oracle's model outputs by 0.4 % shows the same ordering (DDIM max 1.3-2.6 against p 0.6-1.5): the
    deterministic chain of random weights carries an eps difference further than the ancestral one, whose fresh noise
    is shared by both runs. The maximum is a single-element statistic of that process and is not bounded; the rms
    and the 99.9th percentile are, at ~1.5x the worst emulated case. A wrong table row or update moves the rms to ~1."""
    d = (mel.float().cpu() - ref.float().cpu()).abs().flatten()
    mx, rms = d.max().item(), d.pow(2).mean().sqrt().item()
    q = d.kthvalue(max(1, int(0.999 * d.numel()))).values.item()
    assert rms < 0.4 and q < 6.0, (what, mx, q, rms)
    return mx, q, rms


def test_engine_on_emulation_matches_golden(gold, emu):
    """DiffusionEngine.sample(sampler="ddim") on the emulated kernel library against the reference's DDIM loop
    (check_ddim_mel). Changing eta refills the tables of the same workspace."""
    from tortoise_tts_b200.diffusion_engine import DiffusionEngine
    cfg = ModelConfig.small()
    eng = DiffusionEngine(synth_all(cfg, seed=0, suppress_stop=False)["diffusion"], cfg, device="cpu")
    st = None
    for case in gold["cases"]:
        n = case["iters"]
        mel = eng.sample(gold["latents"][0], gold["cond"][0], n, gold["noise0"][0], gold["step_noise"][:n, 0],
                         cond_free=case["cond_free"], cond_free_k=gold["cond_free_k"], use_graph=False,
                         sampler="ddim", eta=case["eta"])
        check_ddim_mel(mel, case["mel"][0], (case["iters"], case["eta"], case["cond_free"]))
        if case["iters"] == 6 and case["cond_free"]:
            assert st is None or eng._ws is st, "a new eta allocated a new workspace"
            st = eng._ws


def _bare_facade():
    from tortoise_tts_b200.api import TextToSpeech
    return TextToSpeech.__new__(TextToSpeech)        # no models: the checks must come before any work


@pytest.mark.parametrize("kw", [dict(diffusion_sampler="x"), dict(ddim_eta=-0.1), dict(ddim_eta=1.5),
                                dict(diffusion_sampler="ddim", ddim_eta=1.5), dict(diffusion_sampler="ddim",
                                                                                   ddim_eta=float("nan"))])
def test_facade_rejects_bad_sampler_arguments(kw):
    t = _bare_facade()
    with pytest.raises(ValueError):
        t.tts("hello", **kw)
    with pytest.raises(ValueError):
        t.tts_with_preset("hello", preset="ultra_fast", **kw)
    with pytest.raises(ValueError):
        t.tts_batch(["hello", "there"], preset="ultra_fast", **kw)
    with pytest.raises(ValueError):
        t.tts_long("hello|there", preset="ultra_fast", **kw)


def test_engine_rejects_bad_sampler_arguments():
    from tortoise_tts_b200.diffusion_engine import DiffusionEngine
    eng = DiffusionEngine.__new__(DiffusionEngine)
    eng.C, eng.dev = 64, torch.device("cpu")
    lat, n0 = torch.zeros(10, 8), torch.zeros(100, 43)
    for kw in (dict(sampler="x"), dict(sampler="ddim", eta=1.5), dict(sampler="ddim", eta=-0.1)):
        with pytest.raises(ValueError):
            eng.sample(lat, torch.zeros(128), 4, n0, torch.zeros(4, 100, 43), **kw)


def _pair_worker(rank, ws, port):
    """The CFG branches split over a rank pair with the all-gather fallback (gloo here), DDIM epilogue on both ranks."""
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import tortoise_tts_b200.lib as real
    from tortoise_tts_b200 import parallel
    from tortoise_tts_b200.diffusion_engine import DiffusionEngine
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=ws)
    try:
        lib_emu.install()
        real.ddim_step = ddim_step
        cfg = ModelConfig.small()
        sd = synth_all(cfg, seed=0, suppress_stop=False)["diffusion"]
        g = torch.Generator().manual_seed(5)
        N, iters = 8, 3
        S = N * 4 * 24000 // 22050
        lat, cond = torch.randn(N, cfg.ar_dim, generator=g), torch.randn(2 * cfg.diff_dim, generator=g) * 0.3
        n0, sn = torch.randn(100, S, generator=g), torch.randn(iters, 100, S, generator=g)
        groups, _ = parallel.pair_groups()
        kw = dict(cond_free=True, cond_free_k=2.0, use_graph=False, sampler="ddim", eta=0.5)
        mel_pair = DiffusionEngine(sd, cfg, device="cpu").sample(lat, cond, iters, n0, sn, pair=(groups[0], rank), **kw)
        mel_one = DiffusionEngine(sd, cfg, device="cpu").sample(lat, cond, iters, n0, sn, **kw)
        assert (mel_pair - mel_one).abs().max().item() < 1e-4
    finally:
        dist.destroy_process_group()


def test_cfg_pair_split_world2_ddim():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    mp.spawn(_pair_worker, args=(2, port), nprocs=2, join=True)
