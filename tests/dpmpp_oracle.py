"""TEST INFRASTRUCTURE ONLY (CPU oracle) — DPM-Solver++(2M) (Lu et al. 2022, arXiv:2211.01095, Algorithm 2: the
multistep second-order solver in data prediction, as k-diffusion's sample_dpmpp_2m runs it) over oracle/diffusion.py's
respaced schedule and DiffusionTts forward. The reference has no such sampler, so this restates the paper: it is written
in the paper's terms (alpha, sigma and lambda of each spaced index, x0 predictions) from float64 scalars, not from the
engine's table rows. order=1 drops the multistep correction, which makes it DDIM at eta = 0. Never imported by the
product path."""
import numpy as np
import torch

from oracle import diffusion as od


def respaced_alphas_cumprod(iters, trained_steps=4000):
    """(alphas_cumprod float64 [n], timestep_map int64 [n]) of od.make_schedule's respaced schedule, read off the base
    schedule at the kept timesteps (od.make_schedule itself needs 2 steps for its posterior tables)."""
    scale = 1000 / trained_steps
    base_ac = np.cumprod(1.0 - np.linspace(scale * 0.0001, scale * 0.02, trained_steps, dtype=np.float64))
    use = np.array(od.space_timesteps_single(trained_steps, iters), dtype=np.int64)
    return base_ac[use], use


def dpmpp_schedule(iters):
    """float64 numpy arrays indexed by the spaced step i: alpha, sigma, lam of i and of its target i - 1 (the target of
    i = 0 has sigma = 0, lam = +inf), the eps -> x0 factors, and the timestep map."""
    ac, tmap = respaced_alphas_cumprod(iters)
    ac_prev = np.append(1.0, ac[:-1])
    alpha, sigma = np.sqrt(ac), np.sqrt(1.0 - ac)
    lam = np.log(alpha) - np.log(sigma)
    return {"alpha": alpha, "sigma": sigma, "lam": lam, "alpha_prev": np.sqrt(ac_prev),
            "sigma_prev": np.sqrt(1.0 - ac_prev), "lam_prev": np.append(np.inf, lam[:-1]),
            "sqrt_recip_ac": np.sqrt(1.0 / ac), "sqrt_recipm1_ac": np.sqrt(1.0 / ac - 1), "timestep_map": tmap}


def dpmpp_update(sch, i, n, x, eps, eps_u, x0_prev, cond_free_k=2.0, order=2):
    """One call at spaced step i of n after the model call: x, eps (conditional), eps_u (unconditional or None) and
    x0_prev (the previous call's x0; unused on the first call) -> (x', x0). The learned-variance half plays no part.
    The arithmetic runs in x's dtype with float64 coefficients."""
    if eps_u is not None:
        cfk = cond_free_k * (1 - i / n)
        eps = (1 + cfk) * eps - cfk * eps_u
    x0 = (float(sch["sqrt_recip_ac"][i]) * x - float(sch["sqrt_recipm1_ac"][i]) * eps).clamp(-1, 1)
    if i == 0:
        return x0, x0           # the step to sigma = 0 returns the data prediction (sample_dpmpp_2m at sigma_next = 0)
    h = float(sch["lam_prev"][i] - sch["lam"][i])
    d = x0
    if order == 2 and i < n - 1:
        r = float(sch["lam"][i] - sch["lam"][i + 1]) / h       # previous call's step over this one
        d = (1 + 1 / (2 * r)) * x0 - (1 / (2 * r)) * x0_prev
    x_new = float(sch["sigma_prev"][i] / sch["sigma"][i]) * x - float(sch["alpha_prev"][i] * np.expm1(-h)) * d
    return x_new, x0


def sample(model, x, iters, cond_free_k=2.0, order=2):
    """The solver loop from the injected x_T = x. model(x, i) -> (eps, eps_u or None) at spaced step i. Returns x_0."""
    sch = dpmpp_schedule(iters)
    n = len(sch["timestep_map"])
    x0_prev = None
    for i in reversed(range(n)):
        eps, eps_u = model(x, i)
        x, x0_prev = dpmpp_update(sch, i, n, x, eps, eps_u, x0_prev, cond_free_k, order)
    return x


def dpmpp_sample_loop(sd, cfg, code_emb, noise0, iters, cond_free=True, cond_free_k=2.0, order=2):
    """The solver on the DiffusionTts oracle, in the convention of od.p_sample_loop: noise0 [1, 100, S] is x_T. The
    solver draws no noise. Returns x_0 [1, 100, S]."""
    tmap = respaced_alphas_cumprod(iters)[1]
    cin = cfg.diff_in_channels

    def model(x, i):
        t_orig = torch.tensor([int(tmap[i])], dtype=torch.long)
        eps = od.forward(sd, cfg, x, t_orig, code_emb=code_emb)[:, :cin]
        eps_u = od.forward(sd, cfg, x, t_orig, conditioning_free=True)[:, :cin] if cond_free else None
        return eps, eps_u
    return sample(model, noise0, iters, cond_free_k, order)
