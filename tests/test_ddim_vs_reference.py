"""Pins the DDIM oracle (tests/ddim_oracle.py) and make_ddim_schedule against the UNMODIFIED reference's
SpacedDiffusion (the copy build() places under oracle/_ref; without it these tests skip and
tests/golden/ddim_small_v1.pt carries the pin instead)."""
import numpy as np
import pytest
import torch

import ddim_oracle
from tortoise_tts_b200.config import ModelConfig
from tortoise_tts_b200.diffusion_engine import make_ddim_schedule
from tortoise_tts_b200.synth import synth_all

pytestmark = pytest.mark.reference


@pytest.fixture(scope="module")
def small():
    from oracle.ref_build import build_reference_models
    cfg = ModelConfig.small()
    sds = synth_all(cfg, seed=0, suppress_stop=False)
    with torch.no_grad():
        dm = build_reference_models(cfg, sds, kv_cache=True)["diffusion"]
    return cfg, sds["diffusion"], dm


@pytest.mark.parametrize("cond_free", [True, False])
@pytest.mark.parametrize("eta", [0.0, 0.5, 1.0])
@pytest.mark.parametrize("iters", [2, 5, 30])        # the reference cannot build a one-step schedule (diffusion.py:240)
def test_ddim_loop_matches_reference(small, iters, eta, cond_free):
    """oracle ddim_sample_loop == load_discrete_vocoder_diffuser(...).ddim_sample_loop under the same torch RNG stream
    (x_T, then one randn_like per step, drawn even at eta = 0). At 2 steps and eta = 1 the reference's fp32
    sqrt(1 - ac_prev - sigma^2) takes the root of a radicand rounded below 0 and returns NaN; the oracle follows it
    there (make_ddim_schedule does not: test_ddim_schedule_kats)."""
    from tortoise.api import load_discrete_vocoder_diffuser
    cfg, sd, dm = small
    torch.manual_seed(11)
    N = 8
    S = N * 4 * 24000 // 22050
    lat = torch.randn(1, N, cfg.ar_dim)
    cond = torch.randn(1, 2 * cfg.diff_dim) * 0.3
    with torch.no_grad():
        ce = dm.timestep_independent(lat, cond, S, False)
        diffuser = load_discrete_vocoder_diffuser(desired_diffusion_steps=iters, cond_free=cond_free, cond_free_k=2.0)
        torch.manual_seed(12)
        noise0 = torch.randn(1, 100, S)
        want = diffuser.ddim_sample_loop(dm, (1, 100, S), noise=noise0,
                                         model_kwargs={"precomputed_aligned_embeddings": ce}, progress=False, eta=eta)
        torch.manual_seed(12)
        noise0 = torch.randn(1, 100, S)
        step_noise = torch.stack([torch.randn(1, 100, S) for _ in range(iters)])
        got = ddim_oracle.ddim_sample_loop(sd, cfg, ce, noise0, step_noise, iters, eta, cond_free, 2.0)
    assert torch.equal(torch.isnan(got), torch.isnan(want))
    ok = ~torch.isnan(want)
    if ok.any():
        assert (got[ok] - want[ok]).abs().max().item() < 1e-3


@pytest.mark.parametrize("eta", [0.0, 0.3, 1.0])
def test_ddim_schedule_kats(eta):
    """make_ddim_schedule rows against the reference's alphas_cumprod / alphas_cumprod_prev arrays: the first three are
    the float64 arrays rounded once; sigma and dir agree with the reference's fp32 torch expressions to fp32 rounding."""
    from oracle.ref_shims import load_reference
    load_reference()
    from tortoise.api import load_discrete_vocoder_diffuser
    for iters in (2, 5, 30, 200):
        d = load_discrete_vocoder_diffuser(desired_diffusion_steps=iters)
        tmap, tb = make_ddim_schedule(iters, eta)
        assert tb.dtype == np.float32 and tb.shape == (5, len(d.timestep_map))
        assert list(tmap) == list(d.timestep_map)
        assert np.array_equal(tb[0], d.sqrt_recip_alphas_cumprod.astype(np.float32))
        assert np.array_equal(tb[1], d.sqrt_recipm1_alphas_cumprod.astype(np.float32))
        assert np.array_equal(tb[2], np.sqrt(d.alphas_cumprod_prev).astype(np.float32))
        ab, abp = d.alphas_cumprod, d.alphas_cumprod_prev
        sigma = eta * np.sqrt((1 - abp) / (1 - ab)) * np.sqrt(1 - ab / abp)
        assert np.allclose(tb[4], sigma, rtol=1e-6, atol=0)
        assert np.allclose(tb[3], np.sqrt(np.maximum(0, 1 - abp - sigma ** 2)), rtol=1e-6, atol=0)
        # the reference's own fp32 expressions (utils/diffusion.py:654-666) lose digits in 1 - ab / abp and in the
        # radicand, which it may round below 0 (NaN) at eta = 1
        abf, abpf = torch.from_numpy(ab).float(), torch.from_numpy(abp).float()
        sig32 = eta * torch.sqrt((1 - abpf) / (1 - abf)) * torch.sqrt(1 - abf / abpf)
        dir32 = torch.sqrt(1 - abpf - sig32 ** 2).numpy()
        assert np.abs(tb[4] - sig32.numpy()).max() < 1e-5
        fin = np.isfinite(dir32)
        assert np.abs(tb[3][fin] - dir32[fin]).max() < 1e-4
        assert tb[3][0] == 0.0 and tb[4][0] == 0.0              # the last step returns x0 itself
        assert (tb[3] >= 0).all() and np.isfinite(tb).all()
