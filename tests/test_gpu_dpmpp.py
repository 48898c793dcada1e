"""GPU: the DPM-Solver++(2M) sampler (ttb_dpmpp2m_step, DiffusionEngine.sample(sampler="dpm++2m"),
tts(diffusion_sampler="dpm++2m")).

The kernel against a float64 numpy step; the engine on the small checkpoint against the oracle loop
(tests/dpmpp_oracle.py) from the same x_T; the full-size denoiser at S = 1872; the facade against the engine on the
captured latents and x_T; the CFG pair on two GPUs against one GPU."""
import os
import socket

import numpy as np
import pytest
import torch

from gpu_util import report
from test_dpmpp_host import _oracle_mel, check_dpmpp_mel, mel_stats

pytestmark = pytest.mark.gpu
MEL_MAX, MEL_MIN = 2.3143386840820312, -11.512925148010254


def _step64(tb, i, iters, x, eps, eps_u, x0_prev, cond_free_k):
    """The 2M update in float64 on the fp32 table values the kernel reads -> (x', D, the magnitude of D's operands)."""
    t = tb.astype(np.float64)[:, i]
    if eps_u is not None:
        cfk = cond_free_k * (1 - i / iters)
        eps = (1 + cfk) * eps - cfk * eps_u
    d = np.clip(t[0] * x - t[1] * eps, -1, 1)
    dm = t[4] * d + (t[5] * x0_prev if t[5] != 0 else 0.0)
    return t[2] * x + t[3] * dm, d, np.abs(t[0] * x).max() + np.abs(t[1] * eps).max()


@pytest.mark.parametrize("parity", [False, True])
@pytest.mark.parametrize("cond_free", [True, False])
def test_dpmpp2m_step_kernel(cond_free, parity):
    """ttb_dpmpp2m_step at the first, a middle and the last call against float64, bound fp32 rounding (1e-5 of
    max(1, |x'|)); x0_prev after the call holds D, the bf16 copy is x' rounded, the mel is written on the last call
    only. On the first and the last call x0_prev starts NaN-filled and must not leak into x'. `parity` lays model_out
    out as the double-buffered peer-exchange area (parity_stride) of the two-GPU CFG pair, with the other slot NaN."""
    from tortoise_tts_b200 import lib
    from tortoise_tts_b200.diffusion_engine import make_dpmpp2m_schedule
    dev = "cuda"
    iters, S, C, ld_xb = 30, 37, 100, 128
    _, tables = make_dpmpp2m_schedule(iters)
    g = torch.Generator().manual_seed(7)
    x_init = torch.randn(S, C, generator=g) * 3
    mo = torch.randn(2, S, 2 * C, generator=g)
    prev = torch.rand(S, C, generator=g) * 2 - 1
    n = S * 2 * C
    worst = 0.0
    for call in (0, 13, iters - 1):
        i = iters - 1 - call
        if parity:
            area = torch.full((2, 2 * n), float("nan"))
            area[call & 1] = mo.reshape(-1)
            model_out, stride = area.to(dev), 2 * n
        else:
            model_out, stride = mo.to(dev), 0
        x = x_init.to(dev, copy=True)
        first_order = tables[5, i] == 0
        assert first_order == (call in (0, iters - 1))
        x0p = torch.full((S, C), float("nan")) if first_order else prev.clone()
        x0p = x0p.to(dev)
        xb = torch.zeros(S, ld_xb, dtype=torch.bfloat16, device=dev)
        mel = torch.full((C, S), 123.0, device=dev)
        lib.dpmpp2m_step(model_out, n, 2 * C, x, xb, ld_xb, torch.from_numpy(tables).to(dev),
                         torch.tensor([call], dtype=torch.int32, device=dev), S, C, iters, cond_free, 2.0, x0p, mel,
                         parity_stride=stride)
        want, d, d_scale = _step64(tables, i, iters, x_init.double().numpy(), mo[0, :, :C].double().numpy(),
                                   mo[1, :, :C].double().numpy() if cond_free else None, prev.double().numpy(), 2.0)
        got = x.cpu().double().numpy()
        assert np.isfinite(got).all()
        err = np.abs(got - want).max() / max(1.0, np.abs(want).max())
        worst = max(worst, err)
        assert err < 1e-5, (call, err)
        # D = sqrt_recip_ac x - sqrt_recipm1_ac eps cancels (both factors ~150 on the first call): its fp32 error is
        # relative to the operands
        assert np.abs(x0p.cpu().double().numpy() - d).max() < 1e-6 * max(1.0, d_scale), call
        assert torch.equal(xb[:, :C].cpu(), x.cpu().to(torch.bfloat16))
        assert (xb[:, C:] == 0).all()
        if i == 0:
            assert np.abs(want).max() <= 1.0
            assert torch.allclose(mel.cpu(), ((x.cpu() + 1) / 2 * (MEL_MAX - MEL_MIN) + MEL_MIN).t(), atol=1e-5)
        else:
            assert (mel == 123.0).all()
    report("dpmpp2m_step kernel vs float64 cf=%d parity=%d (rel)" % (cond_free, parity), worst)


@pytest.fixture(scope="module")
def small():
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_all
    cfg = ModelConfig.small()
    return cfg, synth_all(cfg, seed=0, suppress_stop=False)


def test_engine_small_vs_oracle(small):
    """The engine against the oracle loop from the same x_T (check_dpmpp_mel, derived from the emulated drift; the
    2-call chain is reported, see there), CFG on and off and 1 to 8 steps; graph and eager agree bit for bit; the
    default sampler is still the p sampler."""
    from tortoise_tts_b200.diffusion_engine import DiffusionEngine
    cfg, sds = small
    sd = sds["diffusion"]
    eng = DiffusionEngine(sd, cfg)
    g = torch.Generator().manual_seed(8)
    N = 9
    S = N * 4 * 24000 // 22050
    lat, cond = torch.randn(N, cfg.ar_dim, generator=g), torch.randn(2 * cfg.diff_dim, generator=g) * 0.3
    n0 = torch.randn(100, S, generator=g)
    for n, cf in ((8, True), (6, True), (4, False), (3, True), (2, True), (1, True)):
        sn = torch.randn(n, 100, S, generator=g)
        kw = dict(cond_free=cf, cond_free_k=2.0, sampler="dpm++2m")
        eager = eng.sample(lat, cond, n, n0, sn, use_graph=False, **kw).cpu()
        graph = eng.sample(lat, cond, n, n0, sn, **kw).cpu()
        d = (eager - graph).abs().max().item()
        report("dpm++2m small graph vs eager iters=%d cf=%d" % (n, cf), d)
        assert torch.equal(eager, graph), d
        ref = _oracle_mel(sd, cfg, lat, cond, n0, n, cf)
        mx, q, rms = mel_stats(graph, ref) if n == 2 else check_dpmpp_mel(graph, ref, (n, cf))
        assert torch.isfinite(graph).all()
        name = "dpm++2m small vs oracle iters=%d cf=%d" % (n, cf)
        report("%s max (range 13.8)" % name, mx)
        report("%s p99.9" % name, q)
        report("%s rms" % name, rms)
    # deterministic given x_T: the step noises are not read
    sn = torch.randn(8, 100, S, generator=g)
    a = eng.sample(lat, cond, 8, n0, sn, sampler="dpm++2m")
    b = eng.sample(lat, cond, 8, n0, torch.randn(8, 100, S, generator=g), sampler="dpm++2m")
    assert torch.equal(a, b)
    p0 = eng.sample(lat, cond, 8, n0, sn)
    p1 = eng.sample(lat, cond, 8, n0, sn, sampler="p")
    assert torch.equal(p0, p1)
    assert not torch.equal(p0, a)


def test_engine_full_size_s1872():
    """ModelConfig.full() synthetic denoiser, S = 1872, 20 steps: graph replay and the eager loop agree bit for bit, and
    the mel is finite and inside the denormalised range (the last call returns the clamped x0)."""
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.diffusion_engine import DiffusionEngine
    from tortoise_tts_b200.synth import synth_diffusion
    cfg = ModelConfig.full()
    eng = DiffusionEngine(synth_diffusion(cfg, seed=3), cfg)
    g = torch.Generator().manual_seed(9)
    N, n = 430, 20
    S = N * 4 * 24000 // 22050
    assert S == 1872
    lat, cond = torch.randn(N, cfg.ar_dim, generator=g), torch.randn(2 * cfg.diff_dim, generator=g) * 0.3
    n0, sn = torch.randn(100, S, generator=g), torch.randn(n, 100, S, generator=g)
    graph = eng.sample(lat, cond, n, n0, sn, sampler="dpm++2m").cpu()
    eager = eng.sample(lat, cond, n, n0, sn, sampler="dpm++2m", use_graph=False).cpu()
    replay = eng.sample(lat, cond, n, n0, sn, sampler="dpm++2m").cpu()
    report("dpm++2m full S=1872 graph vs eager", (graph - eager).abs().max().item())
    assert torch.equal(graph, eager)
    assert torch.equal(graph, replay)
    assert graph.shape == (100, S) and torch.isfinite(graph).all()
    assert graph.min().item() >= MEL_MIN - 1e-4 and graph.max().item() <= MEL_MAX + 1e-4
    report("dpm++2m full S=1872 mel range", graph.max().item() - graph.min().item())


def _facade(small):
    from tortoise_tts_b200.api import TextToSpeech
    cfg, sds = small
    return TextToSpeech(state_dicts=sds, config=cfg, enable_redaction=False)


def test_facade_tts_dpmpp_equals_engine(small):
    cfg, _ = small
    tts = _facade(small)
    toks = [42, 2, 194, 91, 24, 2, 243, 190, 2, 182, 37, 2]
    g = torch.Generator().manual_seed(4)
    cl = (torch.randn(1, cfg.ar_dim, generator=g), torch.randn(1, 2 * cfg.diff_dim, generator=g) * 0.3)
    kw = dict(text_tokens=toks, conditioning_latents=cl, use_deterministic_seed=5, max_mel_tokens=24,
              num_autoregressive_samples=8, diffusion_iterations=8, verbose=False)
    tts.debug_capture = True
    w = tts.tts("unused", diffusion_sampler="dpm++2m", ddim_eta=0.4, **kw)
    dbg = tts.last_debug
    tts.debug_capture = False
    assert w.shape[:2] == (1, 1) and torch.isfinite(w).all()
    noise0, step_noise = dbg["noise"][0]
    want = tts.diffusion.sample(dbg["latents"][0], cl[1].cuda().float().reshape(-1), 8, noise0, step_noise,
                                cond_free=True, cond_free_k=2, sampler="dpm++2m")
    assert torch.equal(dbg["mel"][0], want)
    # ddim_eta is ignored by this sampler; the default is the p sampler; every sampler starts from the same x_T
    w0 = tts.tts("unused", diffusion_sampler="dpm++2m", **kw)
    assert torch.equal(w, w0)
    tts.debug_capture = True
    a = tts.tts("unused", **kw)
    assert torch.equal(tts.last_debug["noise"][0][0], noise0)
    tts.debug_capture = False
    assert not torch.equal(a, w)


def test_facade_tts_batch_dpmpp_equals_tts_per_text(small):
    """The setup under which test_gpu_tts_batch.py asserts tts_batch == tts per text (mixed step, one warp per stream),
    with the 2M sampler."""
    from tortoise_tts_b200 import ar_engine
    cfg, _ = small
    tts = _facade(small)
    torch.manual_seed(5)
    toks = [torch.randint(1, 255, (n,)).tolist() for n in (12, 30, 7)]
    g = torch.Generator().manual_seed(6)
    cond = (torch.randn(1, cfg.ar_dim, generator=g), torch.randn(1, 2 * cfg.diff_dim, generator=g))
    kw = dict(conditioning_latents=cond, use_deterministic_seed=3, max_mel_tokens=40, num_autoregressive_samples=6,
              diffusion_iterations=5, diffusion_sampler="dpm++2m")
    E = ar_engine.AREngine
    saved = E.MODE
    os.environ["TTB_AR_STEP_TEAM"] = "1"
    try:
        E.MODE = "mixed"
        got = tts.tts_batch(["x"] * 3, preset="ultra_fast", text_tokens_list=toks, **kw)
        for u in range(3):
            want = tts.tts_with_preset("x", preset="ultra_fast", text_tokens=toks[u], **kw)
            assert got[u].shape == want.shape
            d = (got[u] - want).abs().max().item()
            report("tts_batch dpm++2m vs tts waveform u=%d" % u, d)
            assert d == 0.0
    finally:
        E.MODE = saved
        os.environ.pop("TTB_AR_STEP_TEAM", None)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _pair_worker(rank, ws, port):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=ws, device_id=torch.device("cuda", rank))
    try:
        from tortoise_tts_b200 import parallel
        from tortoise_tts_b200.config import ModelConfig
        from tortoise_tts_b200.diffusion_engine import DiffusionEngine
        from tortoise_tts_b200.synth import synth_all
        cfg = ModelConfig.small()
        sd = synth_all(cfg, seed=0, suppress_stop=False)["diffusion"]
        g = torch.Generator().manual_seed(5)
        N, n = 12, 6
        S = N * 4 * 24000 // 22050
        lat, cond = torch.randn(N, cfg.ar_dim, generator=g), torch.randn(2 * cfg.diff_dim, generator=g) * 0.3
        n0, sn = torch.randn(100, S, generator=g), torch.randn(n, 100, S, generator=g)
        groups, npairs = parallel.pair_groups()
        assert npairs == 1
        pair = DiffusionEngine(sd, cfg).sample(lat, cond, n, n0, sn, sampler="dpm++2m", pair=(groups[0], rank))
        one = DiffusionEngine(sd, cfg).sample(lat, cond, n, n0, sn, sampler="dpm++2m")
        # each rank evaluates one branch with the kernels that evaluate it in the batch of two
        assert (pair - one).abs().max().item() < 1e-3, rank
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="the CFG pair needs 2 GPUs")
def test_cfg_pair_two_gpus_dpmpp():
    import torch.multiprocessing as mp
    mp.spawn(_pair_worker, args=(2, _free_port()), nprocs=2, join=True)
