#!/usr/bin/env python
"""CPU study (not a test): error of ONE denoiser evaluation (eps/variance prediction, both CFG branches) when the
conv / attention GEMM operands are rounded to bf16 (the engine today) or to FP8 e4m3 (per-tensor scale for weights,
per-token scale for activations). FP8 operands would halve the bytes the TMA has to deliver per k-block;
the parity bound on this check is 3 %.
Run: python tests/study_gemm_precision.py"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from oracle import diffusion as od  # noqa: E402
from tortoise_tts_b200.config import ModelConfig  # noqa: E402
from tortoise_tts_b200.synth import synth_all  # noqa: E402


def r_bf16(t, dim=None):
    return t.to(torch.bfloat16).float()


def r_fp8(t, dim):
    """e4m3 with a scale per slice along `dim` (None = one scale for the tensor)."""
    s = (t.abs().amax() if dim is None else t.abs().amax(dim=dim, keepdim=True)).clamp_min(1e-12) / 448.0
    return (t / s).to(torch.float8_e4m3fn).float() * s


def patched(round_act, round_w):
    real_conv, real_einsum = F.conv1d, torch.einsum

    def conv1d(x, w, b=None, **kw):
        # x [B, C, T]: activations are token-major in the engine -> one scale per token (dim=1); weights per tensor
        return real_conv(round_act(x, 1), round_w(w, None), b, **kw)

    def einsum(eq, a, b):
        return real_einsum(eq, round_act(a, 1), round_act(b, 1))
    return conv1d, einsum


def main():
    cfg = ModelConfig.full()
    sd = synth_all(cfg, seed=0, suppress_stop=True)["diffusion"]
    g = torch.Generator().manual_seed(1)
    S = 374
    x = torch.randn(1, 100, S, generator=g)
    ce = torch.randn(1, cfg.diff_dim, S, generator=g)
    t = torch.tensor([3979])
    with torch.no_grad():
        ref = od.forward(sd, cfg, x, t, code_emb=ce)
        print("one denoiser forward at full width, S=%d; output scale %.3f" % (S, ref.abs().max().item()))
        for name, (ra, rw) in {"bf16 operands (engine today)": (r_bf16, r_bf16),
                               "fp8 weights, bf16 activations": (r_bf16, r_fp8),
                               "fp8 weights + fp8 activations (per-token scale)": (r_fp8, r_fp8)}.items():
            real = (F.conv1d, torch.einsum)
            F.conv1d, torch.einsum = patched(ra, rw)
            try:
                got = od.forward(sd, cfg, x, t, code_emb=ce)
            finally:
                F.conv1d, torch.einsum = real
            print("  %-48s rel err (max|d| / max|ref|) %.4f   rms %.5f" %
                  (name, (got - ref).abs().max().item() / ref.abs().max().item(),
                   (got - ref).pow(2).mean().sqrt().item() / ref.abs().max().item()))


if __name__ == "__main__":
    main()
