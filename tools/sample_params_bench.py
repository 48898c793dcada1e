"""Cost of sampling every row with its own settings (ttb_ar_sample_params) against the scalar sampler, on the full-size
synthetic checkpoint (stop token suppressed, streams decode to their cap). Three measurements in one run:
  sampler  - ttb_ar_sample against ttb_ar_sample_params with equal settings, V = 8194, B in --batch; CUDA events over
             --launches launches per arm, --rounds rounds with the arms alternated; min and max per launch;
  batch    - tts_stream_batch of 32 and 128 texts without kwargs_list and with a kwargs_list of identical settings: the
             tokens must be identical; decode device time per step;
  pool     - the 32-listener arrival trace of tools/stream_pool_bench.py (one every --every-ms, seeded jitter) into a
             fresh pool of 32 slots per run: every stream with the pool's settings (the scalar sampler), then every
             stream with its own (the per-row sampler from the first admission on): wait to the first chunk
             p50 / p95 / max and underruns.
Reads the GPU's name, power limit and SM clock. Prints one JSON line.

    python tools/sample_params_bench.py [--rounds 3] [--launches 2000]
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from fast_batch_bench import gpu_state  # noqa: E402
from stream_pool_bench import summarize  # noqa: E402

V, STOP = 8194, 8193
MIXED = [dict(temperature=0.6, top_p=0.9), dict(top_k=7, repetition_penalty=1.5), dict(temperature=1.2, top_k=20),
         dict(top_p=0.5, repetition_penalty=3.0)]


def sampler(lib, B, launches, rounds):
    g = torch.Generator().manual_seed(B)
    logits = (torch.randn(B, V, generator=g) * 3).cuda()
    u = torch.rand(B, 4, generator=g).cuda()
    seen = torch.zeros(B, (V + 31) // 32, dtype=torch.int32, device="cuda")
    codes = torch.zeros(B, 4, dtype=torch.int32, device="cuda")
    fin = torch.zeros(B, dtype=torch.int32, device="cuda")
    state = torch.zeros(64, dtype=torch.int32, device="cuda")
    table = lib.sample_params_table([dict(temperature=0.8, top_k=50, top_p=0.8, repetition_penalty=2.0)] * B, "cuda")
    arms = {"scalar": lambda: lib.ar_sample(logits, V, V, B, u, 4, seen, codes, 4, fin, state, 0.8, 50, 0.8, 2.0, STOP,
                                            advance=False),
            "per_row": lambda: lib.ar_sample_params(logits, V, V, B, u, 4, seen, codes, 4, fin, state, table, STOP,
                                                    advance=False)}
    res = {k: [] for k in arms}
    for f in arms.values():
        for _ in range(50):
            f()
    for _ in range(rounds):
        for k, f in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(launches):
                f()
            e1.record()
            e1.synchronize()
            res[k].append(e0.elapsed_time(e1) * 1e3 / launches)
    return {k: [round(min(v), 2), round(max(v), 2)] for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 16, 64, 128, 256])
    ap.add_argument("--launches", type=int, default=2000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--streams", type=int, nargs="+", default=[32, 128])
    ap.add_argument("--listeners", type=int, default=32)
    ap.add_argument("--every-ms", type=float, default=250.0)
    ap.add_argument("--chunk", type=int, default=40)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sample_params_bench needs a CUDA device")
    from tortoise_tts_b200 import api_fast, lib
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_autoregressive, synth_hifigan, synth_rlg
    res = {"gpu_before": gpu_state()}
    res["sampler_us_per_launch"] = {B: sampler(lib, B, args.launches, args.rounds) for B in args.batch}

    cfg = ModelConfig()
    sds = {"autoregressive": synth_autoregressive(cfg, 0, True), "hifigan": synth_hifigan(cfg, 0),
           "rlg_auto": synth_rlg(cfg.ar_dim, 0)}
    tts = api_fast.TextToSpeech(state_dicts=sds, config=cfg, kv_cache=True)
    kw = dict(verbose=False, stream_chunk_size=args.chunk, use_deterministic_seed=1)
    g = torch.Generator().manual_seed(0)
    batch = {}
    for R in args.streams:
        toks = [torch.randint(1, 255, (n,), generator=g).tolist() for n in torch.randint(40, 91, (R,), generator=g)]
        same = [dict(temperature=0.8, top_p=0.8, top_k=50, repetition_penalty=2.0)] * R
        arm_ms, codes = {}, {}
        for rnd in range(args.rounds + 1):                       # round 0 warms up both graphs
            for name, kl in (("scalar", None), ("kwargs_list", same)):
                box = {}
                real = tts.autoregressive.generate_grouped_stream

                def rec(*a, **k):
                    for y in real(*a, **k):
                        box["codes"] = [c.clone() for c in y[0]]
                        yield y
                tts.autoregressive.generate_grouped_stream = rec
                for _ in tts.tts_stream_batch(["x"] * R, text_tokens_list=toks, kwargs_list=kl, **kw):
                    pass
                del tts.autoregressive.generate_grouped_stream
                steps = max(tts.last_timings["tokens"])
                if rnd:
                    arm_ms.setdefault(name, []).append(tts.last_timings["ar_ms"] / steps)
                codes[name] = box["codes"]
        same_tokens = all(torch.equal(a, b) for a, b in zip(codes["scalar"], codes["kwargs_list"]))
        batch[R] = {k: [round(min(v), 3), round(max(v), 3)] for k, v in arm_ms.items()}
        batch[R]["identical_tokens"] = same_tokens
    res["stream_batch_decode_ms_per_step"] = batch

    N = args.listeners
    lens = torch.randint(40, 91, (N,), generator=g).tolist()
    toks = [torch.randint(1, 255, (n,), generator=g).tolist() for n in lens]
    jit = (torch.rand(N, generator=g) - 0.5).tolist()
    arrive = sorted(max(0.0, (u + jit[u]) * args.every_ms / 1e3) for u in range(N))

    def run_pool(settings):
        pool = tts.stream_pool(max_streams=32, verbose=False, stream_chunk_size=args.chunk)
        arr, sid_u, nxt = [[] for _ in range(N)], {}, 0
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        while True:
            now = time.perf_counter() - t0
            while nxt < N and arrive[nxt] <= now:
                sid_u[pool.submit("x", text_tokens=toks[nxt], use_deterministic_seed=1 + nxt, **settings(nxt))] = nxt
                nxt += 1
            ev = pool.poll()
            if not ev:
                if nxt == N:
                    break
                time.sleep(max(0.0, arrive[nxt] - (time.perf_counter() - t0)))
                continue
            torch.cuda.synchronize()
            t = time.perf_counter() - t0
            for sid, chunk, last in ev:
                arr[sid_u[sid]].append((t, int(chunk.numel())))
        wall = time.perf_counter() - t0
        per_row = bool(pool.ws.sp.get("per_row"))
        pool.close()
        out = summarize(arr, arrive, wall, {})
        return {**{k: round(out[k], 1) for k in ("wait_p50_ms", "wait_p95_ms", "wait_max_ms", "underruns")},
                "per_row_sampler": per_row}

    arms = {"uniform": lambda u: {}, "mixed": lambda u: MIXED[u % len(MIXED)]}
    res["pool_32_listeners"] = {k: [] for k in arms}
    for rnd in range(args.rounds + 1):                             # round 0 warms up both arms
        for k, f in arms.items():
            r = run_pool(f)
            if rnd:
                res["pool_32_listeners"][k].append(r)
    res["gpu_after"] = gpu_state()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
