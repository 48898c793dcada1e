"""Times api_fast.TextToSpeech.tts_batch against a loop of api_fast tts() calls over the same sentences (full-size
synthetic checkpoint, stop token suppressed, so every sentence decodes `max_mel_tokens - 1` tokens). Seeded token lists
of 40-90 tokens; the loop arm runs over the largest count once per round and its first n sentences give the loop time
of n sentences (each tts() call is independent of the others). Rounds alternate the arms. Device stage times come from
CUDA events (`last_timings`), wall times from a host clock around calls that end in a device synchronise. The GPU's
name, power limit and SM clock are read in the same run. Prints one JSON line.

    python tools/fast_batch_bench.py [--sizes 64 128] [--rounds 3] [--max-mel-tokens 604]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_state():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = "nvidia-smi unavailable: %s" % e
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[64, 128])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--max-mel-tokens", type=int, default=604, help="model limit: every sentence decodes this - 1")
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fast_batch_bench needs a CUDA device")
    from tortoise_tts_b200 import api_fast
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_autoregressive, synth_hifigan, synth_rlg
    cfg = ModelConfig(max_mel_tokens=args.max_mel_tokens)
    sds = {"autoregressive": synth_autoregressive(cfg, 0, True), "hifigan": synth_hifigan(cfg, 0),
           "rlg_auto": synth_rlg(cfg.ar_dim, 0)}
    tts = api_fast.TextToSpeech(state_dicts=sds, config=cfg, kv_cache=True)
    n_all = max(args.sizes)
    g = torch.Generator().manual_seed(args.seed)
    lens = torch.randint(40, 91, (n_all,), generator=g).tolist()
    toks = [torch.randint(1, 255, (n,), generator=g).tolist() for n in lens]
    kw = dict(use_deterministic_seed=1, verbose=False)
    res = {"gpu_before": gpu_state(), "max_mel_tokens": args.max_mel_tokens, "text_tokens": [min(lens), max(lens)],
           "sizes": args.sizes, "rounds": args.rounds}

    def run_batch(n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        wavs = tts.tts_batch(["x"] * n, text_tokens_list=toks[:n], **kw)
        samples = sum(int(w.numel()) for w in wavs)
        t1 = time.perf_counter()
        tim = dict(tts.last_timings)
        tim.pop("tokens")
        return {"wall_ms": (t1 - t0) * 1e3, "audio_s": samples / 24000.0,
                "audio_s_per_s": samples / 24000.0 / (t1 - t0), **tim}, [int(w.numel()) for w in wavs]

    def run_loop():
        per = []
        for u in range(n_all):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            w = tts.tts("x", text_tokens=toks[u], **kw)
            n = int(w.numel())
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            per.append(dict(wall_ms=(t1 - t0) * 1e3, samples=n, **{k: v for k, v in tts.last_timings.items()
                                                                     if k.endswith("_ms")}))
        out = {}
        for n in args.sizes:
            s = per[:n]
            wall = sum(p["wall_ms"] for p in s)
            samples = sum(p["samples"] for p in s)
            out[n] = {"wall_ms": wall, "audio_s": samples / 24000.0, "audio_s_per_s": samples / 24000.0 / (wall / 1e3),
                      **{k: sum(p[k] for p in s) for k in ("ar_ms", "latents_ms", "hifigan_ms")}}
        return out, [p["samples"] for p in per]

    # warm-up: modules, graphs of the one-row step, both batch sizes
    tts.tts("x", text_tokens=toks[0], **kw)
    for n in args.sizes:
        run_batch(n)
    rounds = []
    for r in range(args.rounds):
        loop, loop_len = run_loop()
        batch = {}
        for n in args.sizes:
            batch[n], blen = run_batch(n)
            assert blen == loop_len[:n], "waveform lengths differ between the arms"
        rounds.append({"loop": loop, "batch": batch})
    res["rounds_data"] = rounds
    summ = {}
    for n in args.sizes:
        for arm in ("loop", "batch"):
            keys = [k for k in rounds[0][arm][n] if k.endswith("_ms") or k == "audio_s_per_s"]
            summ["%s_%d" % (arm, n)] = {k: [round(min(rd[arm][n][k] for rd in rounds), 1),
                                            round(max(rd[arm][n][k] for rd in rounds), 1)] for k in keys}
        summ["speedup_wall_%d" % n] = [round(min(rd["loop"][n]["wall_ms"] / rd["batch"][n]["wall_ms"] for rd in rounds), 2),
                                      round(max(rd["loop"][n]["wall_ms"] / rd["batch"][n]["wall_ms"] for rd in rounds), 2)]
    res["summary_min_max"] = summ
    res["gpu_after"] = gpu_state()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
