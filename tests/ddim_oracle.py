"""TEST INFRASTRUCTURE ONLY (CPU oracle) — restatement of SpacedDiffusion.ddim_sample_loop (utils/diffusion.py:623-793)
over oracle/diffusion.py's schedule and DiffusionTts forward: p_mean_variance (CFG ramp, eps -> x0, clamp), eps
re-derived from the clamped x0 (_predict_eps_from_xstart, 437-441), then eq. 12 with sigma(eta). The per-step arithmetic
is fp32 torch on fp32-extracted tables, as the reference's _extract_into_tensor gives it. Never imported by the product
path."""
import numpy as np
import torch

from oracle import diffusion as od


def ddim_tables(iters):
    """fp32 tensors of the tables ddim_sample reads, indexed by the spaced step i, and the timestep map."""
    sch = od.make_schedule(iters)
    ac = sch["alphas_cumprod"]
    f32 = {"sqrt_recip_ac": sch["sqrt_recip_alphas_cumprod"], "sqrt_recipm1_ac": sch["sqrt_recipm1_alphas_cumprod"],
           "ac": ac, "ac_prev": np.append(1.0, ac[:-1])}
    return {k: torch.from_numpy(v.astype(np.float32)) for k, v in f32.items()}, sch["timestep_map"]


def ddim_update(tb, i, n, x, eps, eps_u, noise, eta, cond_free_k):
    """One ddim_sample update after the model call at spaced step i of n: x, eps (conditional), eps_u (unconditional
    or None), noise -> x'. The learned-variance half of the model output plays no part."""
    if eps_u is not None:
        cfk = cond_free_k * (1 - i / n)
        eps = (1 + cfk) * eps - cfk * eps_u
    x0 = (tb["sqrt_recip_ac"][i] * x - tb["sqrt_recipm1_ac"][i] * eps).clamp(-1, 1)
    eps = (tb["sqrt_recip_ac"][i] * x - x0) / tb["sqrt_recipm1_ac"][i]
    ab, abp = tb["ac"][i], tb["ac_prev"][i]
    sigma = eta * torch.sqrt((1 - abp) / (1 - ab)) * torch.sqrt(1 - ab / abp)
    mean = x0 * torch.sqrt(abp) + torch.sqrt(1 - abp - sigma ** 2) * eps
    nz = 0.0 if i == 0 else 1.0
    return mean + nz * sigma * noise


def ddim_sample_loop(sd, cfg, code_emb, noise0, step_noise, iters, eta, cond_free=True, cond_free_k=2.0):
    """SpacedDiffusion.ddim_sample_loop with injected randomness, in the convention of od.p_sample_loop: noise0
    [1, 100, S] is x_T; ddim_sample draws randn_like on EVERY step (even at eta = 0), and the draw of call c is
    step_noise[c] ([iters, 1, 100, S]). Returns x_0 [1, 100, S]."""
    tb, tmap = ddim_tables(iters)
    n = len(tmap)
    cin = cfg.diff_in_channels
    x = noise0
    for call, i in enumerate(reversed(range(n))):
        t_orig = torch.tensor([int(tmap[i])], dtype=torch.long)
        eps = od.forward(sd, cfg, x, t_orig, code_emb=code_emb)[:, :cin]
        eps_u = od.forward(sd, cfg, x, t_orig, conditioning_free=True)[:, :cin] if cond_free else None
        x = ddim_update(tb, i, n, x, eps, eps_u, step_noise[call], eta, cond_free_k)
    return x
