"""Cost of the typical-set filter (typical_sampling=True) on one GPU, with CUDA events:

  * the sampler kernel alone, ttb_ar_sample against ttb_ar_sample_typical (mass 0.9), at B = 128 and 256, V = 8194,
    over many launches after a warm-up (advance = 0, so every launch samples the same step);
  * the whole AR stage of the standard workload (bench.py's configs[2]: full-size synthetic checkpoint, 256 candidates,
    the para53 paragraph, 430 mel tokens), filter off and on, alternated.

Prints one JSON line with the GPU's name and power limit. Needs a CUDA device (there is no CPU fallback)."""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _gpu():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def kernel_us(lib, B, mass, launches=500, warmup=50):
    V = 8194
    g = torch.Generator(device="cuda").manual_seed(B)
    logits = torch.randn(B, V, device="cuda", generator=g) * 3
    u = torch.rand(B, 1, device="cuda", generator=g)
    seen = torch.zeros(B, (V + 31) // 32, dtype=torch.int32, device="cuda")
    seen[:, 0] = 2
    codes = torch.empty(B, 1, dtype=torch.int32, device="cuda")
    fin = torch.zeros(B, dtype=torch.int32, device="cuda")
    state = torch.zeros(64, dtype=torch.int32, device="cuda")

    def run():
        if mass is None:
            lib.ar_sample(logits, V, V, B, u, 1, seen, codes, 1, fin, state, 0.8, 50, 0.8, 2.0, 8193, advance=False)
        else:
            lib.ar_sample_typical(logits, V, V, B, u, 1, seen, codes, 1, fin, state, 0.8, 50, 0.8, 2.0, 8193, mass,
                                  advance=False)
    for _ in range(warmup):
        run()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    ev[0].record()
    for _ in range(launches):
        run()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) * 1e3 / launches


def main(rounds=3, mass=0.9):
    if not torch.cuda.is_available():
        raise SystemExit("typical_bench needs a CUDA device")
    import __graft_entry__ as ge
    ge.build()
    from tortoise_tts_b200 import lib
    from tortoise_tts_b200.ar_engine import AREngine
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_all
    out = {"gpu": _gpu(), "typical_mass": mass, "kernel_us": {}}
    for B in (128, 256):
        off = [kernel_us(lib, B, None) for _ in range(rounds)]
        on = [kernel_us(lib, B, mass) for _ in range(rounds)]
        out["kernel_us"]["B=%d" % B] = {"off": sorted(off)[rounds // 2], "on": sorted(on)[rounds // 2]}
    with open(os.path.join(ROOT, "tests", "golden", "bench_text_tokens.json")) as f:
        tokens = json.load(f)["para53"]["tokens"]
    cfg = ModelConfig.full()
    eng = AREngine(synth_all(cfg, seed=0, suppress_stop=True)["autoregressive"], cfg)
    g = torch.Generator().manual_seed(0)
    cond = (torch.randn(1, cfg.ar_dim, generator=g) * 0.5).reshape(-1).cuda()
    toks = [int(t) for t in tokens] + [0]
    B, N = 256, 430
    u = torch.rand(B, N, generator=torch.Generator().manual_seed(1)).cuda()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    times = {"off": [], "on": []}
    steps = {}
    for r in range(rounds + 1):                 # round 0 warms up (graph capture for each setting)
        for name, m in (("off", None), ("on", mass)):
            torch.cuda.synchronize()
            ev[0].record()
            codes = eng.generate(cond, toks, B, N, uniforms=u, typical_mass=m)
            ev[1].record()
            torch.cuda.synchronize()
            if r:
                times[name].append(ev[0].elapsed_time(ev[1]))
            steps[name] = int((codes != cfg.stop_mel_token).sum(1).max().item())
    out["ar_stage_ms"] = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    out["ar_stage_all_ms"] = times
    out["ar_longest_candidate_tokens"] = steps
    out["ar_workload"] = "configs[2] AR stage: 256 candidates, %d-token paragraph, max %d mel tokens" % (len(tokens), N)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
