"""GPU: the DDIM sampler (ttb_ddim_step, DiffusionEngine.sample(sampler="ddim"), tts(diffusion_sampler="ddim")).

The kernel against a float64 numpy step; the engine on the small checkpoint against the DDIM oracle and the reference's
loop (tests/golden/ddim_small_v1.pt) with the same injected noise; the full-size denoiser at S = 1872; the facade against
the engine on the captured latents and noise; the CFG pair on two GPUs against one GPU."""
import os
import socket

import numpy as np
import pytest
import torch

import ddim_oracle
from gpu_util import report
from test_ddim_host import check_ddim_mel

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "ddim_small_v1.pt")
MEL_MAX, MEL_MIN = 2.3143386840820312, -11.512925148010254


def _step64(tb, i, iters, x, eps, eps_u, noise, cond_free_k):
    """The DDIM update in float64 on the fp32 table values the kernel reads."""
    t = tb.astype(np.float64)[:, i]
    if eps_u is not None:
        cfk = cond_free_k * (1 - i / iters)
        eps = (1 + cfk) * eps - cfk * eps_u
    x0 = np.clip(t[0] * x - t[1] * eps, -1, 1)
    e2 = (t[0] * x - x0) / t[1]
    nz = 0.0 if i == 0 else 1.0
    return t[2] * x0 + t[3] * e2 + nz * t[4] * (0.0 if noise is None else noise)


@pytest.mark.parametrize("parity", [False, True])
@pytest.mark.parametrize("eta", [0.0, 0.7])
@pytest.mark.parametrize("cond_free", [True, False])
def test_ddim_step_kernel(cond_free, eta, parity):
    """ttb_ddim_step at the first, a middle and the last call (mel written) against float64, bound fp32 rounding
    (1e-5 of max(1, |x'|)). eta = 0 runs with noise = NULL. `parity` lays model_out out as the double-buffered
    peer-exchange area (parity_stride) of the two-GPU CFG pair, with the other slot holding garbage."""
    from tortoise_tts_b200 import lib
    from tortoise_tts_b200.diffusion_engine import make_ddim_schedule
    dev = "cuda"
    iters, S, C, ld_xb = 30, 37, 100, 128
    _, tables = make_ddim_schedule(iters, eta)
    tb = torch.zeros(6, iters)                       # the engine's table buffer has 6 rows; DDIM reads the first 5
    tb[:5] = torch.from_numpy(tables)
    g = torch.Generator().manual_seed(7)
    x_init = torch.randn(S, C, generator=g) * 3
    mo = torch.randn(2, S, 2 * C, generator=g)
    noise = torch.randn(iters, S, C, generator=g) if eta > 0 else None
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
        x = x_init.to(dev)
        xb = torch.zeros(S, ld_xb, dtype=torch.bfloat16, device=dev)
        mel = torch.full((C, S), 123.0, device=dev)
        lib.ddim_step(model_out, n, 2 * C, x, xb, ld_xb, None if noise is None else noise.to(dev), tb.to(dev),
                      torch.tensor([call], dtype=torch.int32, device=dev), S, C, iters, cond_free, 2.0, mel,
                      parity_stride=stride)
        want = _step64(tables, i, iters, x_init.double().numpy(), mo[0, :, :C].double().numpy(),
                       mo[1, :, :C].double().numpy() if cond_free else None,
                       None if noise is None else noise[call].double().numpy(), 2.0)
        got = x.cpu().double().numpy()
        err = np.abs(got - want).max() / max(1.0, np.abs(want).max())
        worst = max(worst, err)
        assert err < 1e-5, (call, err)
        assert torch.equal(xb[:, :C].cpu(), x.cpu().to(torch.bfloat16))
        assert (xb[:, C:] == 0).all()
        if i == 0:
            assert np.abs(want).max() <= 1.0
            assert torch.allclose(mel.cpu(), ((x.cpu() + 1) / 2 * (MEL_MAX - MEL_MIN) + MEL_MIN).t(), atol=1e-5)
        else:
            assert (mel == 123.0).all()
    report("ddim_step kernel vs float64 cf=%d eta=%.1f parity=%d (rel)" % (cond_free, eta, parity), worst)


@pytest.fixture(scope="module")
def small():
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_all
    cfg = ModelConfig.small()
    return cfg, synth_all(cfg, seed=0, suppress_stop=False)


def _stats(name, mel, ref):
    mx, q, rms = check_ddim_mel(mel, ref, name)
    report("%s max (range 13.8)" % name, mx)
    report("%s p99.9" % name, q)
    report("%s rms" % name, rms)


def test_engine_small_vs_golden_and_oracle(small):
    from tortoise_tts_b200.diffusion_engine import DiffusionEngine
    from oracle import diffusion as od
    cfg, sds = small
    gold = torch.load(GOLD)
    eng = DiffusionEngine(sds["diffusion"], cfg)
    lat, cond = gold["latents"][0], gold["cond"][0]
    for case in gold["cases"]:
        n = case["iters"]
        kw = dict(cond_free=case["cond_free"], cond_free_k=gold["cond_free_k"], sampler="ddim", eta=case["eta"])
        mels = [eng.sample(lat, cond, n, gold["noise0"][0], gold["step_noise"][:n, 0], use_graph=ug, **kw).cpu()
                for ug in (False, True)]
        _stats("ddim small vs reference iters=%d eta=%.1f cf=%d" % (n, case["eta"], case["cond_free"]), mels[1],
               case["mel"][0])
        d = (mels[0] - mels[1]).abs().max().item()
        report("ddim small graph vs eager iters=%d eta=%.1f" % (n, case["eta"]), d)
        assert d < 1e-3
    # a chain the fixture does not hold, against the oracle run here
    g = torch.Generator().manual_seed(8)
    N, n, eta = 9, 8, 0.3
    S = N * 4 * 24000 // 22050
    lat2, cond2 = torch.randn(N, cfg.ar_dim, generator=g), torch.randn(2 * cfg.diff_dim, generator=g) * 0.3
    n0, sn = torch.randn(100, S, generator=g), torch.randn(n, 100, S, generator=g)
    with torch.no_grad():
        ce = od.timestep_independent(sds["diffusion"], cfg, lat2.unsqueeze(0), cond2.unsqueeze(0), S)
        want = od.denormalize_tacotron_mel(ddim_oracle.ddim_sample_loop(sds["diffusion"], cfg, ce, n0.unsqueeze(0),
                                                                         sn.unsqueeze(1), n, eta, True, 2.0))[0]
    got = eng.sample(lat2, cond2, n, n0, sn, sampler="ddim", eta=eta).cpu()
    _stats("ddim small vs oracle iters=8 eta=0.3", got, want)
    # eta = 0 is deterministic; the default sampler is the p sampler, bit for bit
    a = eng.sample(lat2, cond2, n, n0, sn, sampler="ddim", eta=0.0)
    b = eng.sample(lat2, cond2, n, n0, sn, sampler="ddim", eta=0.0)
    assert torch.equal(a, b)
    p0 = eng.sample(lat2, cond2, n, n0, sn)
    p1 = eng.sample(lat2, cond2, n, n0, sn, sampler="p")
    assert torch.equal(p0, p1)
    assert not torch.equal(p0, a)


def test_engine_full_size_s1872():
    """ModelConfig.full() synthetic denoiser, S = 1872, 50 DDIM steps: finite, inside the denormalised range (the last
    step returns the clamped x0), and a new eta replays the captured graph instead of capturing another."""
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.diffusion_engine import DiffusionEngine
    from tortoise_tts_b200.synth import synth_diffusion
    cfg = ModelConfig.full()
    eng = DiffusionEngine(synth_diffusion(cfg, seed=3), cfg)
    g = torch.Generator().manual_seed(9)
    N, n = 430, 50
    S = N * 4 * 24000 // 22050
    assert S == 1872
    lat, cond = torch.randn(N, cfg.ar_dim, generator=g), torch.randn(2 * cfg.diff_dim, generator=g) * 0.3
    n0, sn = torch.randn(100, S, generator=g), torch.randn(n, 100, S, generator=g)
    graph = None
    for eta in (0.0, 0.5, 1.0):
        mel = eng.sample(lat, cond, n, n0, sn, sampler="ddim", eta=eta).cpu()
        assert mel.shape == (100, S) and torch.isfinite(mel).all()
        assert mel.min().item() >= MEL_MIN - 1e-4 and mel.max().item() <= MEL_MAX + 1e-4
        if graph is None:
            graph = eng._ws["graph"]
        assert eng._ws["graph"] is graph, "a new eta captured a new graph"
        report("ddim full S=1872 eta=%.1f mel range" % eta, mel.max().item() - mel.min().item())


def _facade(small):
    from tortoise_tts_b200.api import TextToSpeech
    cfg, sds = small
    return TextToSpeech(state_dicts=sds, config=cfg, enable_redaction=False)


def test_facade_tts_ddim_equals_engine(small):
    cfg, _ = small
    tts = _facade(small)
    toks = [42, 2, 194, 91, 24, 2, 243, 190, 2, 182, 37, 2]
    g = torch.Generator().manual_seed(4)
    cl = (torch.randn(1, cfg.ar_dim, generator=g), torch.randn(1, 2 * cfg.diff_dim, generator=g) * 0.3)
    kw = dict(text_tokens=toks, conditioning_latents=cl, use_deterministic_seed=5, max_mel_tokens=24,
              num_autoregressive_samples=8, diffusion_iterations=8, verbose=False)
    tts.debug_capture = True
    w = tts.tts("unused", diffusion_sampler="ddim", ddim_eta=0.4, **kw)
    dbg = tts.last_debug
    tts.debug_capture = False
    assert w.shape[:2] == (1, 1) and torch.isfinite(w).all()
    noise0, step_noise = dbg["noise"][0]
    want = tts.diffusion.sample(dbg["latents"][0], cl[1].cuda().float().reshape(-1), 8, noise0, step_noise,
                                cond_free=True, cond_free_k=2, sampler="ddim", eta=0.4)
    assert torch.equal(dbg["mel"][0], want)
    # the default is the p sampler, and both samplers start from the same x_T and vocoder noise
    a = tts.tts("unused", **kw)
    tts.debug_capture = True
    b = tts.tts("unused", diffusion_sampler="p", **kw)
    assert torch.equal(tts.last_debug["noise"][0][0], noise0)
    tts.debug_capture = False
    assert torch.equal(a, b)
    assert not torch.equal(a, w)


def test_facade_tts_batch_ddim_equals_tts_per_text(small):
    """The setup under which test_gpu_tts_batch.py asserts tts_batch == tts per text (mixed step, one warp per stream),
    with the DDIM sampler."""
    from tortoise_tts_b200 import ar_engine
    cfg, _ = small
    tts = _facade(small)
    torch.manual_seed(5)
    toks = [torch.randint(1, 255, (n,)).tolist() for n in (12, 30, 7)]
    g = torch.Generator().manual_seed(6)
    cond = (torch.randn(1, cfg.ar_dim, generator=g), torch.randn(1, 2 * cfg.diff_dim, generator=g))
    kw = dict(conditioning_latents=cond, use_deterministic_seed=3, max_mel_tokens=40, num_autoregressive_samples=6,
              diffusion_iterations=4, diffusion_sampler="ddim", ddim_eta=0.5)
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
            report("tts_batch ddim vs tts waveform u=%d" % u, d)
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
        for eta in (0.0, 0.6):
            pair = DiffusionEngine(sd, cfg).sample(lat, cond, n, n0, sn, sampler="ddim", eta=eta, pair=(groups[0], rank))
            one = DiffusionEngine(sd, cfg).sample(lat, cond, n, n0, sn, sampler="ddim", eta=eta)
            # each rank evaluates one branch with the kernels that evaluate it in the batch of two
            assert (pair - one).abs().max().item() < 1e-3, (rank, eta)
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="the CFG pair needs 2 GPUs")
def test_cfg_pair_two_gpus_ddim():
    import torch.multiprocessing as mp
    mp.spawn(_pair_worker, args=(2, _free_port()), nprocs=2, join=True)
