"""Device time of the diffusion stage with the p sampler, with DDIM and with DPM-Solver++(2M), on one GPU, with CUDA
events.

The stage is DiffusionEngine.sample as tts() runs it (timestep-independent conditioning, tables, noise upload and every
captured step, both CFG branches) on the full-size synthetic checkpoint at S = 1872 (430 latents, the length of the
standard benchmark's utterance): p at 200 steps, DDIM (eta = 0) at 200, 100, 50 and 25 steps, DPM-Solver++(2M) at 50,
25, 20 and 10 steps. Every arm is captured and warmed first; the timed rounds alternate the arms. The SM clock is read
while the last round runs.

Prints one JSON line with the GPU's name, power limit and SM clock. Needs a CUDA device (there is no CPU fallback)."""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ARMS = [("p", 200), ("ddim", 200), ("ddim", 100), ("ddim", 50), ("ddim", 25),
        ("dpm++2m", 50), ("dpm++2m", 25), ("dpm++2m", 20), ("dpm++2m", 10)]
QUERY = ["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"]


def main(rounds=3):
    if not torch.cuda.is_available():
        raise SystemExit("ddim_bench needs a CUDA device")
    import __graft_entry__ as ge
    ge.build()
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.diffusion_engine import DiffusionEngine
    from tortoise_tts_b200.synth import synth_diffusion
    cfg = ModelConfig.full()
    sd = synth_diffusion(cfg, seed=3)
    # one engine per arm: an engine keeps the workspace and graph of its last (S, steps, sampler) only
    engines = {a: DiffusionEngine(sd, cfg) for a in ARMS}
    g = torch.Generator().manual_seed(0)
    N = 430
    S = N * 4 * 24000 // 22050
    lat, cond = torch.randn(N, cfg.ar_dim, generator=g), torch.randn(2 * cfg.diff_dim, generator=g) * 0.3
    n0 = torch.randn(100, S, generator=g)
    noise = {n: torch.randn(n, 100, S, generator=g).cuda() for n in sorted({n for _, n in ARMS})}
    lat, cond, n0 = lat.cuda(), cond.cuda(), n0.cuda()

    def run(sampler, n):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        engines[(sampler, n)].sample(lat, cond, n, n0, noise[n], cond_free=True, cond_free_k=2.0, sampler=sampler)
        ev[1].record()
        ev[1].synchronize()
        return ev[0].elapsed_time(ev[1])

    ms = {a: [] for a in ARMS}
    for a in ARMS:          # capture + warm-up
        run(*a)
        run(*a)
    clock = None
    for r in range(rounds):
        for a in ARMS:
            if r == rounds - 1 and a == ARMS[0]:
                clock = subprocess.Popen(QUERY, stdout=subprocess.PIPE, text=True)
            ms[a].append(run(*a))
    gpu = clock.communicate(timeout=60)[0].strip()
    out = {"gpu": gpu, "S": S, "rounds": rounds, "arms": []}
    for (sampler, n), v in ms.items():
        out["arms"].append({"sampler": sampler, "steps": n, "stage_ms": [round(x, 1) for x in v],
                            "ms_per_step": round(min(v) / n, 3)})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
