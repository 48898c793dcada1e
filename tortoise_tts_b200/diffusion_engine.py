"""DiffusionTts denoiser + SpacedDiffusion sampling loop on the sm_90a kernels (hot loop 2, SURVEY §8 rows a9-a12).

Mirrors `do_spectrogram_diffusion` (tortoise/api.py:117-130): `timestep_independent` once, then `iters` steps of
p_sample (or ddim_sample with `sample(sampler="ddim")`, or DPM-Solver++(2M) with `sample(sampler="dpm++2m")`) with
the conditional and unconditional forward batched as B=2 (the reference runs them sequentially,
utils/diffusion.py:340-342), scheduler tables resident on the device and the whole step captured in one CUDA graph.
Activations are token-major [B, S, C]; convolutions are wgmma GEMMs (k=3 as three shifted TMA loads).
"""
import math

import numpy as np
import torch

from . import lib
from .config import ModelConfig


def _bf(t, dev):
    return t.to(device=dev, dtype=torch.bfloat16).contiguous()


def _f(t, dev):
    return t.to(device=dev, dtype=torch.float32).contiguous()


def _groups_for(C):
    """normalization() rule (arch_util.py:26-41)."""
    groups = 32
    if C <= 16:
        groups = 8
    elif C <= 64:
        groups = 16
    while C % groups != 0:
        groups = int(groups / 2)
    return groups


# ----------------------------------------------------------------------- schedule (host, float64 like the reference)
def _respace(iters, trained_steps):
    """-> (timestep_map int64 [n], betas float64 [n]) of SpacedDiffusion(space_timesteps(trained_steps, [iters]))."""
    scale = 1000 / trained_steps
    base_betas = np.linspace(scale * 0.0001, scale * 0.02, trained_steps, dtype=np.float64)
    base_ac = np.cumprod(1.0 - base_betas, axis=0)
    frac = 1 if iters <= 1 else (trained_steps - 1) / (iters - 1)
    cur, use = 0.0, set()
    for _ in range(iters):
        use.add(round(cur))
        cur += frac
    last, betas, tmap = 1.0, [], []
    for i, ac in enumerate(base_ac):
        if i in use:
            betas.append(1 - ac / last)
            last = ac
            tmap.append(i)
    return np.array(tmap, dtype=np.int64), np.array(betas, dtype=np.float64)


def make_schedule(iters, trained_steps=4000):
    """SpacedDiffusion(space_timesteps(4000,[iters]), linear betas) tables (utils/diffusion.py:94-111,1093-1115,
    1184-1205,192-249). Returns (timestep_map int64[n], tables float32 [6, n])."""
    tmap, betas = _respace(iters, trained_steps)
    alphas = 1.0 - betas
    ac = np.cumprod(alphas, axis=0)
    ac_prev = np.append(1.0, ac[:-1])
    post_var = betas * (1.0 - ac_prev) / (1.0 - ac)
    tables = np.stack([
        np.sqrt(1.0 / ac), np.sqrt(1.0 / ac - 1), np.log(np.append(post_var[1], post_var[1:])), np.log(betas),
        betas * np.sqrt(ac_prev) / (1.0 - ac), (1.0 - ac_prev) * np.sqrt(alphas) / (1.0 - ac)]).astype(np.float32)
    return tmap, tables


def make_ddim_schedule(iters, eta, trained_steps=4000):
    """The tables of ddim_sample (utils/diffusion.py:623-671) on the schedule of make_schedule, built in float64.
    Returns (timestep_map int64 [n], tables float32 [5, n]): sqrt_recip_ac, sqrt_recipm1_ac, sqrt(ac_prev),
    dir = sqrt(max(0, 1 - ac_prev - sigma^2)) and sigma = eta sqrt((1 - ac_prev) / (1 - ac)) sqrt(1 - ac / ac_prev).
    The reference takes the square roots of dir and sigma in fp32 torch; here they are taken in float64 and rounded once,
    so the tables differ from its values by fp32 rounding, and dir's radicand (exactly 0 at the last step) cannot be
    rounded below 0 at eta = 1."""
    tmap, betas = _respace(iters, trained_steps)
    ac = np.cumprod(1.0 - betas, axis=0)
    ac_prev = np.append(1.0, ac[:-1])
    sigma = eta * np.sqrt((1.0 - ac_prev) / (1.0 - ac)) * np.sqrt(1.0 - ac / ac_prev)
    tables = np.stack([np.sqrt(1.0 / ac), np.sqrt(1.0 / ac - 1), np.sqrt(ac_prev),
                       np.sqrt(np.maximum(0.0, 1.0 - ac_prev - sigma ** 2)), sigma]).astype(np.float32)
    return tmap, tables


def make_dpmpp2m_schedule(iters, trained_steps=4000):
    """The tables of the DPM-Solver++(2M) epilogue (Lu et al. 2022, arXiv:2211.01095, Algorithm 2) on the schedule of
    make_schedule, built in float64 and rounded to fp32 once. Returns (timestep_map int64 [n], tables float32 [6, n]):
    sqrt_recip_ac, sqrt_recipm1_ac, a, b, w, w_p. With alpha = sqrt(ac), sigma = sqrt(1 - ac),
    lambda = log(alpha) - log(sigma) and spaced index i stepping to i - 1 (index -1 has ac = 1, lambda = +inf):
    h_i = lambda_{i-1} - lambda_i, a = sigma_{i-1} / sigma_i, b = -alpha_{i-1} expm1(-h_i), r = h_{i+1} / h_i,
    w = 1 + 1 / (2r), w_p = -1 / (2r). The first call (i = n - 1) is first order (w = 1, w_p = 0); the last (i = 0)
    returns x' = D (a = 0, b = 1, w = 1, w_p = 0)."""
    tmap, betas = _respace(iters, trained_steps)
    ac = np.cumprod(1.0 - betas, axis=0)
    ac_prev = np.append(1.0, ac[:-1])
    n = len(tmap)
    lam = 0.5 * (np.log(ac) - np.log(1.0 - ac))
    h = np.full(n, np.inf)
    h[1:] = lam[:-1] - lam[1:]
    a, b = np.zeros(n), np.ones(n)
    a[1:] = np.sqrt((1.0 - ac_prev[1:]) / (1.0 - ac[1:]))
    b[1:] = -np.sqrt(ac_prev[1:]) * np.expm1(-h[1:])
    w, w_p = np.ones(n), np.zeros(n)
    r = h[2:] / h[1:-1]                     # indices 1 .. n-2: the calls between the first and the last
    w[1:-1] = 1.0 + 0.5 / r
    w_p[1:-1] = -0.5 / r
    tables = np.stack([np.sqrt(1.0 / ac), np.sqrt(1.0 / ac - 1), a, b, w, w_p]).astype(np.float32)
    return tmap, tables


def _rel_pos_table(emb_weight, T, scale):
    """RelativePositionBias (xtransformers.py:146-186, bidirectional, 32 buckets, max_distance 64) as a Toeplitz
    table: out[h, r + T - 1] = scale * E[bucket(r), h] for r = k_pos - q_pos in [-(T-1), T-1]."""
    dev = emb_weight.device
    rel = torch.arange(-(T - 1), T, device=dev)
    n = -rel
    nb = 16
    ret = (n < 0).long() * nb
    n = n.abs()
    max_exact = nb // 2
    is_small = n < max_exact
    large = max_exact + (torch.log(n.float() / max_exact) / math.log(64 / max_exact) * (nb - max_exact)).long()
    large = torch.min(large, torch.full_like(large, nb - 1))
    bucket = ret + torch.where(is_small, n, large)
    return (emb_weight[bucket].t().contiguous() * scale).float().contiguous()  # [H, 2T-1]


class _AttnW:
    def __init__(self, sd, p, C, H, dev):
        self.gn_g, self.gn_b = _f(sd[p + "norm.weight"], dev), _f(sd[p + "norm.bias"], dev)
        w = sd[p + "qkv.weight"].reshape(3 * C, C)
        b = sd[p + "qkv.bias"]
        # QKVAttentionLegacy channel order is per head [q(64)|k(64)|v(64)] (arch_util.py:60-63): regroup rows to
        # [q heads | k heads | v heads]
        ch = C // H
        idx = torch.arange(3 * C).reshape(H, 3, ch).permute(1, 0, 2).reshape(-1)
        self.wqkv, self.bqkv = _bf(w[idx], dev), _f(b[idx], dev)
        self.wproj = _bf(sd[p + "proj_out.weight"].reshape(C, C), dev)
        self.bproj = _f(sd[p + "proj_out.bias"], dev)
        key = p + "relative_pos_embeddings.relative_attention_bias.weight"
        self.rel_emb = _f(sd[key], dev) if key in sd else None
        self.rel_scale = float(ch) ** 0.5
        self._tables = {}

    def table(self, T):
        if self.rel_emb is None:
            return None
        if T not in self._tables:
            self._tables[T] = _rel_pos_table(self.rel_emb, T, self.rel_scale)
        return self._tables[T]


class _ResW:
    def __init__(self, sd, p, C, dev):
        self.in_g, self.in_b = _f(sd[p + "in_layers.0.weight"], dev), _f(sd[p + "in_layers.0.bias"], dev)
        self.w_in, self.b_in = _bf(sd[p + "in_layers.2.weight"].reshape(C, C), dev), _f(sd[p + "in_layers.2.bias"], dev)
        self.w_emb, self.b_emb = _f(sd[p + "emb_layers.1.weight"], dev), _f(sd[p + "emb_layers.1.bias"], dev)
        self.out_g, self.out_b = _f(sd[p + "out_layers.0.weight"], dev), _f(sd[p + "out_layers.0.bias"], dev)
        # conv k=3 weight [out, in, 3] -> [out, tap, in] so that K is contiguous per tap
        self.w_out = _bf(sd[p + "out_layers.3.weight"].permute(0, 2, 1).reshape(C, 3 * C), dev)
        self.b_out = _f(sd[p + "out_layers.3.bias"], dev)


def _pad_k(w, kpad):
    """conv weight [out, in, taps] -> [out, taps*kpad] (in zero-padded to kpad)."""
    o, i, t = w.shape
    z = torch.zeros(o, t, kpad, dtype=w.dtype)
    z[:, :, :i] = w.permute(0, 2, 1)
    return z.reshape(o, t * kpad)


class DiffusionEngine:
    def __init__(self, sd, cfg: ModelConfig, device="cuda"):
        self.cfg = cfg
        self.dev = torch.device(device)
        dev = self.dev
        C, H = cfg.diff_dim, cfg.diff_heads
        self.C, self.H = C, H
        self.groups = _groups_for(C)
        self.cin = cfg.diff_in_channels
        self.cin_pad = ((self.cin + 63) // 64) * 64
        self.cout = cfg.diff_out_channels
        self.uncond = _f(sd["unconditioned_embedding"].reshape(C), dev)
        self.w_inp = _bf(_pad_k(sd["inp_block.weight"], self.cin_pad), dev)
        self.b_inp = _f(sd["inp_block.bias"], dev)
        self.te_w0, self.te_b0 = _f(sd["time_embed.0.weight"], dev), _f(sd["time_embed.0.bias"], dev)
        self.te_w2, self.te_b2 = _f(sd["time_embed.2.weight"], dev), _f(sd["time_embed.2.bias"], dev)
        self.code_norm_g, self.code_norm_b = _f(sd["code_norm.weight"], dev), _f(sd["code_norm.bias"], dev)
        Dl = cfg.ar_dim
        self.lat_pad = ((Dl + 63) // 64) * 64
        self.w_latc = _bf(_pad_k(sd["latent_conditioner.0.weight"], self.lat_pad), dev)
        self.b_latc = _f(sd["latent_conditioner.0.bias"], dev)
        self.latc_attn = [_AttnW(sd, f"latent_conditioner.{i}.", C, H, dev) for i in range(1, 5)]
        self.integ = [(_ResW(sd, f"conditioning_timestep_integrator.{i}.resblk.", C, dev),
                       _AttnW(sd, f"conditioning_timestep_integrator.{i}.attn.", C, H, dev)) for i in range(3)]
        self.w_integ = _bf(sd["integrating_conv.weight"].reshape(C, 2 * C), dev)
        self.b_integ = _f(sd["integrating_conv.bias"], dev)
        self.layers = [(_ResW(sd, f"layers.{i}.resblk.", C, dev), _AttnW(sd, f"layers.{i}.attn.", C, H, dev))
                       for i in range(cfg.diff_layers)]
        self.tail = [_ResW(sd, f"layers.{i}.", C, dev) for i in range(cfg.diff_layers, cfg.diff_layers + 3)]
        self.out_g, self.out_b = _f(sd["out.0.weight"], dev), _f(sd["out.0.bias"], dev)
        self.w_outc = _bf(sd["out.2.weight"].permute(0, 2, 1).reshape(self.cout, 3 * C), dev)
        self.b_outc = _f(sd["out.2.bias"], dev)
        self.res_all = [r for r, _ in self.integ] + [r for r, _ in self.layers] + self.tail
        self._ws = None

    # ------------------------------------------------------------------ building blocks on [B, S, C] fp32 (in place)
    def _gn(self, x, B, S, g, b, ws, silu=False, ss=None, ss_row=None, out=None, ready=False):
        """GroupNorm32 (+scale/shift, +SiLU) of x into the bf16 GEMM operand. `ready`: the GEMM that produced x already
        left the statistics in ws['partials'] (see _gnp), so x is read once."""
        fn = lib.groupnorm_apply if ready else lib.groupnorm
        fn(x, B, S, self.C, self.groups, g, b, ws["partials"], scale_shift=ss, ss_bstride=0, ss_row=ss_row,
           ss_row_stride=2 * self.C, silu=silu, out_bf16=ws["a"] if out is None else out, ldo=self.C)

    def _gnp(self, S, ws):
        """kwargs that make a C-wide GEMM leave the GroupNorm statistics of its output for the GroupNorm that follows
        (TtbGemmArgs.gn_partials): 32 channels per group and at most TTB_GROUPNORM_SPLITS row blocks of 32. Otherwise
        the GroupNorm takes its statistics in a separate pass."""
        if self.C == 32 * self.groups and (S + 31) // 32 <= 128:
            return dict(gn_partials=ws["partials"], gn_groups=self.groups)
        return {}

    def _attn_block(self, aw, x, B, S, ws, ready=False):
        """AttentionBlock (arch_util.py:80-123). Returns whether x's GroupNorm statistics are ready for the next block."""
        C, H = self.C, self.H
        gp = self._gnp(S, ws)
        self._gn(x, B, S, aw.gn_g, aw.gn_b, ws, ready=ready)
        # w_static: the C-wide GEMMs of a step put their first weight tiles into the pipeline ahead of
        # griddepcontrol.wait (the GroupNorm in front of them releases its dependents at its start)
        lib.gemm(ws["a"], aw.wqkv, M=S, N=3 * C, K=C, bias=aw.bqkv, out_bf16=ws["qkv"], batch=B, a_bstride=S * C,
                 outb_bstride=S * 3 * C, w_static=True)
        # T5 buckets saturate at max_distance = 64 (xtransformers.py:166-174): |j - i| >= 64 -> constant bias per side
        lib.attention(ws["qkv"], ws["o"], nseq=B, T=S, H=H, ld=3 * C, ldo=C, k_off=C, v_off=2 * C, scale=0.125,
                      bias=aw.table(S), bias_sat=64)
        lib.gemm(ws["o"], aw.wproj, M=S, N=C, K=C, bias=aw.bproj, residual=x, out_f32=x, batch=B, a_bstride=S * C,
                 res_bstride=S * C, outf_bstride=S * C, w_static=True, **gp)
        return bool(gp)

    def _res_block(self, rw, ss, x, B, S, ws, ss_row=None, ready=False):
        """ResBlock (diffusion_decoder.py:60-120); `ready` / return value as in _attn_block."""
        C = self.C
        gp = self._gnp(S, ws)
        self._gn(x, B, S, rw.in_g, rw.in_b, ws, silu=True, ready=ready)
        lib.gemm(ws["a"], rw.w_in, M=S, N=C, K=C, bias=rw.b_in, out_f32=ws["h"], batch=B, a_bstride=S * C,
                 outf_bstride=S * C, w_static=True, **gp)
        self._gn(ws["h"], B, S, rw.out_g, rw.out_b, ws, silu=True, ss=ss, ss_row=ss_row, ready=bool(gp))
        lib.gemm(ws["a"], rw.w_out, M=S, N=C, K=C, taps=3, pad=1, bias=rw.b_out, residual=x, out_f32=x, batch=B,
                 a_bstride=S * C, res_bstride=S * C, outf_bstride=S * C, w_static=True, **gp)
        return bool(gp)

    def _alloc(self, B, S):
        C, dev = self.C, self.dev
        return dict(a=torch.empty(B, S, C, dtype=torch.bfloat16, device=dev),
                    h=torch.empty(B, S, C, dtype=torch.float32, device=dev),
                    qkv=torch.empty(B, S, 3 * C, dtype=torch.bfloat16, device=dev),
                    o=torch.empty(B, S, C, dtype=torch.bfloat16, device=dev),
                    partials=lib.groupnorm_scratch(B, self.groups, dev))

    # ------------------------------------------------------------------ timestep-independent conditioning
    def timestep_independent(self, latents, cond_latent, S):
        """≙ DiffusionTts.timestep_independent (diffusion_decoder.py:232-260). latents [N, ar_dim] fp32,
        cond_latent [2C] -> code_emb fp32 [S, C] (token-major)."""
        C, dev = self.C, self.dev
        N = latents.shape[0]
        ws = self._alloc(1, N)
        lat_bf = torch.zeros(N, self.lat_pad, dtype=torch.bfloat16, device=dev)
        lib.cast_pad_bf16(_f(latents, dev), N, latents.shape[1], latents.shape[1], lat_bf, self.lat_pad)
        x = torch.empty(1, N, C, dtype=torch.float32, device=dev)
        lib.gemm(lat_bf, self.w_latc, M=N, N=C, K=self.lat_pad, taps=3, pad=1, bias=self.b_latc, out_f32=x)
        for aw in self.latc_attn:
            self._attn_block(aw, x, 1, N, ws)
        ss = _f(cond_latent.reshape(-1), dev)  # [scale | shift] (diffusion_decoder.py:237)
        normed = torch.empty(N, C, dtype=torch.float32, device=dev)
        lib.groupnorm(x, 1, N, C, self.groups, self.code_norm_g, self.code_norm_b, ws["partials"], scale_shift=ss,
                      out_f32=normed, ldof=C)
        out = torch.empty(S, C, dtype=torch.float32, device=dev)
        lib.interp_nearest(normed, N, S, C, out_f32=out, ldof=C)
        return out

    # ------------------------------------------------------------------ one denoiser evaluation (both CFG branches)
    def _forward(self, st):
        """DiffusionTts.forward (diffusion_decoder.py:262-322) for batch [cond, uncond] (or one of them) at the timestep
        selected by the device-side call counter, both CFG branches batched in every launch. Writes st['mo_local']
        [B, S, cout]."""
        C, B, S, ws = self.C, st["B"], st["S"], st["ws"]
        xce = st["xce"]
        xce.copy_(st["code_emb_init"])
        rdy = False          # are the GroupNorm statistics of the running activation already in ws["partials"]?
        for j, (rw, aw) in enumerate(self.integ):
            rdy = self._res_block(rw, st["ss_all"][j], xce, B, S, ws, st["counter"], ready=rdy)
            rdy = self._attn_block(aw, xce, B, S, ws, ready=rdy)
        cat = st["cat"]
        # inp_block conv on the shared sample x (a_bstride 0 broadcasts it to both branches); writes cat[..., :C]
        lib.gemm(st["x_bf"], self.w_inp, M=S, N=C, K=self.cin_pad, taps=3, pad=1, bias=self.b_inp, out_bf16=cat, ldob=2 * C,
                 batch=B, a_bstride=0, outb_bstride=S * 2 * C)
        lib.cast_pad_bf16(xce, B * S, C, C, cat[:, :, C:], 2 * C, ncols_out=C)
        x = st["xm"]
        gp = self._gnp(S, ws)
        lib.gemm(cat, self.w_integ, M=S, N=C, K=2 * C, bias=self.b_integ, out_f32=x, batch=B, a_bstride=S * 2 * C,
                 outf_bstride=S * C, **gp)
        rdy = bool(gp)
        n_int = len(self.integ)
        for j, (rw, aw) in enumerate(self.layers):
            rdy = self._res_block(rw, st["ss_all"][n_int + j], x, B, S, ws, st["counter"], ready=rdy)
            rdy = self._attn_block(aw, x, B, S, ws, ready=rdy)
        for j, rw in enumerate(self.tail):
            rdy = self._res_block(rw, st["ss_all"][n_int + len(self.layers) + j], x, B, S, ws, st["counter"], ready=rdy)
        self._gn(x, B, S, self.out_g, self.out_b, ws, silu=True, ready=rdy)
        lib.gemm(ws["a"], self.w_outc, M=S, N=self.cout, K=C, taps=3, pad=1, bias=self.b_outc, out_f32=st["mo_local"],
                 batch=B, a_bstride=S * C, outf_bstride=S * self.cout)

    def _step(self, st):
        self._forward(st)
        self._epilogue(st)

    def _scheduler_step(self, st, model_out, out_bstride, parity_stride=0):
        """The sampler's scheduler epilogue on the model outputs of this call (both CFG branches)."""
        if st["sampler"] == "dpm++2m":
            lib.dpmpp2m_step(model_out, out_bstride, self.cout, st["x"], st["x_bf"], self.cin_pad, st["tables"],
                             st["counter"], st["S"], self.cin, st["iters"], st["cond_free"], st["cond_free_k"],
                             st["x0_prev"], st["mel"], parity_stride=parity_stride)
            return
        step = lib.ddim_step if st["sampler"] == "ddim" else lib.diffusion_step
        step(model_out, out_bstride, self.cout, st["x"], st["x_bf"], self.cin_pad, st["noise"], st["tables"], st["counter"],
             st["S"], self.cin, st["iters"], st["cond_free"], st["cond_free_k"], st["mel"], parity_stride=parity_stride)

    def _epilogue(self, st):
        xch = st.get("xch")
        if xch is not None:
            # CFG pair over peer memory: one captured launch puts my branch into both exchange areas and waits for the
            # partner's (csrc/misc.cu pair_exchange_kernel); the scheduler epilogue then reads the slot of this step's parity
            n = st["S"] * self.cout
            lib.pair_exchange(st["mo_local"], xch.area, xch.peer_area, n, 2 * n, xch.my_idx * n, xch.peer_flags, xch.flags,
                              st["counter"], xch.epoch, xch.done, xch.err)
            self._scheduler_step(st, xch.area, n, parity_stride=2 * n)
            lib.counter_add(st["counter"], 1)
            return
        if st.get("pair") is not None:
            # CFG pair split over 2 GPUs: this rank evaluated ONE branch (rank 0 of the pair = conditional, rank 1 =
            # unconditional); one all-gather of the [S, 200] fp32 outputs (1.5 MB over NVLink) gives both ranks both
            # branches, and both then run the identical scheduler epilogue (same pre-drawn noise) -> no second exchange.
            import torch.distributed as dist
            if st["model_out"].is_cuda:
                dist.all_gather_into_tensor(st["model_out"].view(-1), st["mo_local"].view(-1), group=st["pair"][0])
            else:   # gloo (CPU tests of the host logic)
                dist.all_gather([st["model_out"][0], st["model_out"][1]], st["mo_local"][0], group=st["pair"][0])
        self._scheduler_step(st, st["model_out"], st["S"] * self.cout)
        lib.counter_add(st["counter"], 1)

    def _state(self, S, B, iters, cfk=0.0, pair=None, sampler="p"):
        """B = number of CFG branches evaluated ON THIS RANK (2, or 1 when the pair is split over two GPUs / no CFG).
        The captured graph holds the sampler's epilogue, so the sampler is part of the key; DDIM's eta lives only in
        st['tables']. DPM-Solver++(2M) keeps the previous call's clamped x0 in st['x0_prev'] (per rank)."""
        key = (S, B, iters, cfk, None if pair is None else pair[1], sampler)
        if self._ws is not None and self._ws["key"] == key:
            self._ws["pair"] = pair
            return self._ws
        C, dev = self.C, self.dev
        st = dict(key=key, S=S, B=B, iters=iters, pair=pair, sampler=sampler)
        st["ws"] = self._alloc(B, S)
        st["xce"] = torch.empty(B, S, C, dtype=torch.float32, device=dev)
        st["code_emb_init"] = torch.empty(B, S, C, dtype=torch.float32, device=dev)
        st["cat"] = torch.empty(B, S, 2 * C, dtype=torch.bfloat16, device=dev)
        st["xm"] = torch.empty(B, S, C, dtype=torch.float32, device=dev)
        st["model_out"] = torch.empty(2 if pair is not None else B, S, self.cout, dtype=torch.float32, device=dev)
        st["mo_local"] = torch.empty(1, S, self.cout, dtype=torch.float32, device=dev) if pair is not None else st["model_out"]
        st["x"] = torch.empty(S, self.cin, dtype=torch.float32, device=dev)
        st["x_bf"] = torch.zeros(S, self.cin_pad, dtype=torch.bfloat16, device=dev)
        st["noise"] = torch.empty(iters, S, self.cin, dtype=torch.float32, device=dev)
        st["tables"] = torch.empty(6, iters, dtype=torch.float32, device=dev)
        st["counter"] = torch.zeros(1, dtype=torch.int32, device=dev)
        st["mel"] = torch.empty(self.cin, S, dtype=torch.float32, device=dev)
        st["x0_prev"] = torch.empty(S, self.cin, dtype=torch.float32, device=dev) if sampler == "dpm++2m" else None
        # per-ResBlock [scale | shift] rows for every step, in CALL order; the GroupNorm kernel indexes the row of the
        # current call with the device-side counter, so one captured graph serves every step
        st["ss_all"] = torch.empty(len(self.res_all), iters, 2 * C, dtype=torch.float32, device=dev)
        st["graph"] = None
        st["xch"] = None
        if pair is not None and st["model_out"].is_cuda:
            from . import parallel
            xch = parallel.PairExchange(pair[0], pair[1], S * self.cout, dev)
            st["xch"] = xch if xch.ok else None
        self._ws = st
        return st

    def _prepare_time(self, st, t_list):
        """time_embed(timestep_embedding(t)) and every ResBlock's emb_layers for the given ORIGINAL-scale timesteps
        (one row per call) -> st['ss_all'] [n_res, n, 2C] (diffusion_decoder.py:294, 109-114)."""
        C, dev, n = self.C, self.dev, len(t_list)
        t_call = torch.tensor(t_list, dtype=torch.int32, device=dev)
        te = torch.empty(n, C, dtype=torch.float32, device=dev)
        lib.timestep_embedding(t_call, n, C, te)
        t1 = torch.empty(n, C, dtype=torch.float32, device=dev)
        lib.linear_small(te, n, C, self.te_w0, self.te_b0, C, t1, silu_out=True)
        temb = torch.empty(n, C, dtype=torch.float32, device=dev)
        lib.linear_small(t1, n, C, self.te_w2, self.te_b2, C, temb)
        for j, rw in enumerate(self.res_all):
            lib.linear_small(temb, n, C, rw.w_emb, rw.b_emb, 2 * C, st["ss_all"][j], silu_in=True)

    def forward_once(self, x, t_orig, code_emb):
        """Parity hook ≙ DiffusionTts.forward(x, t, precomputed_aligned_embeddings) and (..., conditioning_free=True)
        (diffusion_decoder.py:262-322): x fp32 [100, S] channel-major, t_orig original-scale timestep, code_emb [S, C].
        Returns (cond_out, uncond_out) fp32 [200, S]."""
        C, dev = self.C, self.dev
        S = x.shape[-1]
        st = self._state(S, 2, 1, -1.0)
        st["code_emb_init"][0].copy_(code_emb)
        lib.broadcast_rows(self.uncond, S, C, st["code_emb_init"][1], None, C)
        self._prepare_time(st, [int(t_orig)])
        lib.transpose_f32(_f(x.reshape(self.cin, S), dev), self.cin, S, st["x"])
        lib.cast_pad_bf16(st["x"], S, self.cin, self.cin, st["x_bf"], self.cin_pad)
        st["counter"].zero_()
        self._forward(st)
        mo = st["model_out"]
        return mo[0].t().contiguous(), mo[1].t().contiguous()

    def sample(self, latents, cond_latent, iters, noise0, step_noise, cond_free=True, cond_free_k=2.0, use_graph=True,
               return_trace=False, pair=None, sampler="p", eta=0.0):
        """≙ do_spectrogram_diffusion (api.py:117-130). latents [N, ar_dim], cond_latent [2C];
        noise0 [100, S] (already scaled by the temperature), step_noise [iters, 100, S] in call order.
        `sampler`: "p" runs p_sample_loop, "ddim" runs ddim_sample_loop with `eta` in [0, 1] (utils/diffusion.py:711-793)
        on the same respaced schedule and model call; DDIM reads step_noise[c] at call c too, scaled by sigma.
        "dpm++2m" runs DPM-Solver++(2M) (make_dpmpp2m_schedule) on the same schedule; it reads no step noise and
        ignores `eta`.
        Returns the denormalised mel fp32 [100, S] (channel-major, as the reference returns it)."""
        C, dev = self.C, self.dev
        N = latents.shape[0]
        S = N * 4 * 24000 // 22050
        # pair = (process group of 2 ranks, my rank in it): the two CFG branches run on two GPUs (see _step)
        if not cond_free:
            pair = None
        B = 1 if (pair is not None or not cond_free) else 2
        if sampler == "p":
            tmap, tables = make_schedule(iters)
        elif sampler == "ddim":
            if not 0.0 <= eta <= 1.0:
                raise ValueError("ddim eta must lie in [0, 1], got %r" % (eta,))
            tmap, tables = make_ddim_schedule(iters, float(eta))
        elif sampler == "dpm++2m":
            tmap, tables = make_dpmpp2m_schedule(iters)
        else:
            raise ValueError("unknown diffusion sampler %r (expected 'p', 'ddim' or 'dpm++2m')" % (sampler,))
        n = len(tmap)
        st = self._state(S, B, n, float(cond_free_k), pair, sampler)
        st["cond_free"], st["cond_free_k"] = bool(cond_free), float(cond_free_k)
        if pair is None or pair[1] == 0:
            code_emb = self.timestep_independent(latents, cond_latent, S)
            st["code_emb_init"][0].copy_(code_emb)
        else:
            lib.broadcast_rows(self.uncond, S, C, st["code_emb_init"][0], None, C)
        if B == 2:
            lib.broadcast_rows(self.uncond, S, C, st["code_emb_init"][1], None, C)
        st["tables"][:tables.shape[0]].copy_(torch.from_numpy(tables))
        # time embeddings of all steps in call order (i = n-1 ... 0), then every ResBlock's emb_layers
        self._prepare_time(st, [int(tmap[n - 1 - c]) for c in range(n)])
        # state: x_T and the pre-drawn noises, token-major
        lib.transpose_f32(_f(noise0.reshape(self.cin, S), dev), self.cin, S, st["x"])
        lib.cast_pad_bf16(st["x"], S, self.cin, self.cin, st["x_bf"], self.cin_pad)
        sn = _f(step_noise.reshape(n, self.cin, S), dev)
        for c in range(n):
            lib.transpose_f32(sn[c], self.cin, S, st["noise"][c])
        st["counter"].zero_()
        trace = []

        # The CUDA graph holds the denoiser evaluation (+ the scheduler epilogue when both CFG branches are local).
        # In pair mode the NCCL all-gather is NOT captured (a capture attempt of torch.distributed collectives dead-locks):
        # graph(forward of my branch) -> eager all-gather -> eager epilogue, per step.
        fused_epilogue = pair is None or st.get("xch") is not None      # the exchange itself is capturable
        if st.get("xch") is not None:
            st["xch"].new_sample()

        def captured():
            if fused_epilogue:
                self._step(st)
            else:
                self._forward(st)

        def after():
            if not fused_epilogue:
                self._epilogue(st)

        def rewind():
            st["counter"].zero_()
            lib.transpose_f32(_f(noise0.reshape(self.cin, S), dev), self.cin, S, st["x"])
            lib.cast_pad_bf16(st["x"], S, self.cin, self.cin, st["x_bf"], self.cin_pad)
        if use_graph and not return_trace:
            if st["graph"] is None:
                captured()  # eager warm-up, then rewind
                after()
                torch.cuda.synchronize()
                rewind()
                if st.get("xch") is not None:
                    st["xch"].new_sample()          # the warm-up step left flags of this epoch behind
                g = torch.cuda.CUDAGraph()
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                c0 = lib.CALLS
                with torch.cuda.stream(side):
                    with torch.cuda.graph(g, stream=side):
                        captured()
                st["graph_calls"] = lib.CALLS - c0
                torch.cuda.current_stream().wait_stream(side)
                st["graph"] = g
                rewind()
            for _ in range(n):
                st["graph"].replay()
                after()
            lib.add_calls(n * st["graph_calls"])
        else:
            for _ in range(n):
                captured()
                after()
                if return_trace:
                    trace.append(st["x"].t().contiguous().clone())
        if st.get("xch") is not None and int(st["xch"].err.item()):
            raise lib.TtbError("CFG pair exchange: the partner rank did not answer within 5 s")
        mel = st["mel"].clone()
        return (mel, trace) if return_trace else mel
