"""Generates tests/golden/ddim_small_v1.pt from the UNMODIFIED reference modules (run where the reference is available:
`python tests/golden/make_ddim_golden.py`). The fixture holds the output of the reference's
SpacedDiffusion.ddim_sample_loop on the synthetic small DiffusionTts (ModelConfig.small(), seed 0) for a few
(iters, eta, cond_free) cases, and its inputs: the latents, the conditioning latent, the precomputed code embedding and
the torch RNG draws the loop consumed (x_T, then one randn_like per step, in call order)."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tortoise_tts_b200.config import ModelConfig  # noqa: E402
from tortoise_tts_b200.synth import synth_all  # noqa: E402
from oracle.ref_build import build_reference_models  # noqa: E402

# (iters, eta, cond_free); every case starts from the same seed, so its draws are a prefix of the stored ones
CASES = [(6, 0.0, True), (6, 0.5, True), (6, 1.0, True), (4, 0.0, False)]
SEED = 91


def main():
    torch.manual_seed(4321)
    cfg = ModelConfig.small()
    sds = synth_all(cfg, seed=0, suppress_stop=False)
    dm = build_reference_models(cfg, sds, kv_cache=True)["diffusion"]
    from tortoise.api import load_discrete_vocoder_diffuser
    from tortoise.utils.audio import denormalize_tacotron_mel
    N = 10
    S = N * 4 * 24000 // 22050
    out = {"weights_checksum": float(sum(v.double().sum() for v in sds["diffusion"].values())), "cond_free_k": 2.0}
    with torch.no_grad():
        lat = torch.randn(1, N, cfg.ar_dim)
        cond = torch.randn(1, 2 * cfg.diff_dim) * 0.3
        ce = dm.timestep_independent(lat, cond, S, False)
        out["latents"], out["cond"], out["code_emb"] = lat, cond, ce
        n_max = max(c[0] for c in CASES)
        torch.manual_seed(SEED)
        out["noise0"] = torch.randn(1, 100, S)
        out["step_noise"] = torch.stack([torch.randn(1, 100, S) for _ in range(n_max)])
        out["cases"] = []
        for iters, eta, cf in CASES:
            diffuser = load_discrete_vocoder_diffuser(desired_diffusion_steps=iters, cond_free=cf, cond_free_k=2.0)
            torch.manual_seed(SEED)
            noise0 = torch.randn(1, 100, S)
            x = diffuser.ddim_sample_loop(dm, (1, 100, S), noise=noise0,
                                          model_kwargs={"precomputed_aligned_embeddings": ce}, progress=False, eta=eta)
            out["cases"].append({"iters": iters, "eta": eta, "cond_free": cf, "x0": x,
                                 "mel": denormalize_tacotron_mel(x)[:, :, :S]})
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ddim_small_v1.pt")
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path) / 1e6, "MB")


if __name__ == "__main__":
    main()
