"""Serves an arrival trace of N listeners (one every --every-ms, seeded jitter of +-50 %) three ways, on the full-size
synthetic checkpoint with the stop token suppressed (every stream decodes to its cap, 500 - prompt positions) and seeded
token lists of 40-90 tokens:
  pool   - TextToSpeech.stream_pool(max_streams=C): a listener is submitted when it arrives and joins the running batch;
  waves  - tts_stream_batch in waves: each batch takes everyone who arrived while the previous one ran;
  loop   - one tts_stream call per listener in arrival order (run only for N <= --loop-streams).
Rounds alternate the arms. Per listener, the wait is measured from its arrival to its first chunk (host clock after a
device synchronise at each chunk); an underrun is a chunk that arrives after the audio before it has finished playing
(24 kHz). Per arm: wait p50 / p95 / max, underruns, audio seconds per second of wall time, and the device time of the
decode (ar_ms), the prefills (prefill_ms) and HiFiGAN (hifigan_ms).

Also, in the same run: the decode step cost of a pool of C slots (prompt capacity 352) against a tts_stream_batch decode
of C short prompts, per step; and the prefill of one admission, the time the running streams are held by it.
Reads the GPU's name, power limit and SM clock. Prints one JSON line.

    python tools/stream_pool_bench.py [--listeners 32] [--every-ms 250] [--capacity 32] [--rounds 3]
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
from stream_batch_bench import listener_stats  # noqa: E402


def pct(v, q):
    v = sorted(v)
    return v[min(len(v) - 1, int(round(q * (len(v) - 1))))]


def summarize(arr, arrive, wall, ms):
    waits, under, audio = [], 0, 0.0
    for a, t_in in zip(arr, arrive):
        t0, u, s = listener_stats(a)
        waits.append(t0 - t_in)
        under += u
        audio += s
    return {"wait_p50_ms": pct(waits, 0.5) * 1e3, "wait_p95_ms": pct(waits, 0.95) * 1e3, "wait_max_ms": max(waits) * 1e3,
            "underruns": under, "audio_s_per_s": audio / wall, "wall_ms": wall * 1e3, **ms}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--listeners", type=int, default=32)
    ap.add_argument("--every-ms", type=float, default=250.0)
    ap.add_argument("--capacity", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--loop-streams", type=int, default=8)
    ap.add_argument("--chunk", type=int, default=40)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("stream_pool_bench needs a CUDA device")
    from tortoise_tts_b200 import api_fast
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_autoregressive, synth_hifigan, synth_rlg
    cfg = ModelConfig()
    sds = {"autoregressive": synth_autoregressive(cfg, 0, True), "hifigan": synth_hifigan(cfg, 0),
           "rlg_auto": synth_rlg(cfg.ar_dim, 0)}
    tts = api_fast.TextToSpeech(state_dicts=sds, config=cfg, kv_cache=True)
    N, C = args.listeners, args.capacity
    g = torch.Generator().manual_seed(args.seed)
    lens = torch.randint(40, 91, (N,), generator=g).tolist()
    toks = [torch.randint(1, 255, (n,), generator=g).tolist() for n in lens]
    jit = (torch.rand(N, generator=g) - 0.5).tolist()
    arrive = [max(0.0, (u + jit[u]) * args.every_ms / 1e3) for u in range(N)]
    arrive.sort()
    kw = dict(verbose=False, stream_chunk_size=args.chunk)
    res = {"gpu_before": gpu_state(), "listeners": N, "every_ms": args.every_ms, "capacity": C,
           "text_tokens": [min(lens), max(lens)], "rounds": args.rounds, "stream_chunk_size": args.chunk}

    def run_pool(pool):
        arr, sid_u, nxt = [[] for _ in range(N)], {}, 0
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        while True:
            now = time.perf_counter() - t0
            while nxt < N and arrive[nxt] <= now:
                sid_u[pool.submit("x", text_tokens=toks[nxt], use_deterministic_seed=1 + nxt)] = nxt
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
        tim = pool.last_timings.values()
        ms = {k: sum(v[k] for v in tim) for k in ("prefill_ms", "hifigan_ms")}
        ms["ar_ms_max_per_stream"] = max(v["ar_ms"] for v in tim)
        pool.last_timings.clear()
        return summarize(arr, arrive, wall, ms)

    def run_waves():
        arr, nxt, ms = [[] for _ in range(N)], 0, {"ar_ms": 0.0, "hifigan_ms": 0.0}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        while nxt < N:
            now = time.perf_counter() - t0
            if arrive[nxt] > now:
                time.sleep(arrive[nxt] - now)
                now = time.perf_counter() - t0
            wave = [u for u in range(nxt, N) if arrive[u] <= now][:256]
            nxt = wave[-1] + 1
            # one seed for a batch: listener u gets the uniforms tts_stream draws for it from seed 1
            for u, chunk, last in tts.tts_stream_batch(["x"] * len(wave), text_tokens_list=[toks[i] for i in wave],
                                                       use_deterministic_seed=1, **kw):
                torch.cuda.synchronize()
                arr[wave[u]].append((time.perf_counter() - t0, int(chunk.numel())))
            for k in ms:
                ms[k] += tts.last_timings[k]
        return summarize(arr, arrive, time.perf_counter() - t0, ms)

    def run_loop():
        arr = [[] for _ in range(N)]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for u in range(N):
            now = time.perf_counter() - t0
            if arrive[u] > now:
                time.sleep(arrive[u] - now)
            for chunk in tts.tts_stream("x", text_tokens=toks[u], use_deterministic_seed=1 + u, **kw):
                torch.cuda.synchronize()
                arr[u].append((time.perf_counter() - t0, int(chunk.numel())))
        return summarize(arr, arrive, time.perf_counter() - t0, {})

    pool = tts.stream_pool(max_streams=C, **kw)
    # warm-up: modules, the pool's step graph, the batch workspaces and the one-row graph
    pool.submit("x", text_tokens=toks[0])
    list(pool.run())
    pool.last_timings.clear()
    list(tts.tts_stream_batch(["x"] * min(N, C), text_tokens_list=toks[:min(N, C)], **kw))
    list(tts.tts_stream("x", text_tokens=toks[0], **kw))
    rounds = []
    for r in range(args.rounds):
        rd = {"pool": run_pool(pool), "waves": run_waves()}
        if N <= args.loop_streams:
            rd["loop"] = run_loop()
        rounds.append(rd)
    res["rounds_data"] = rounds
    res["summary_min_max"] = {arm: {k: [round(min(rd[arm][k] for rd in rounds), 1),
                                        round(max(rd[arm][k] for rd in rounds), 1)] for k in rounds[0][arm]}
                              for arm in rounds[0]}
    if N > args.loop_streams:
        res["summary_min_max"]["loop"] = "not measured"

    # step cost: the pool's graph (C slots, prompt capacity 352) against a grouped decode of C short prompts
    ws = pool.ws
    for s in range(C):
        ws.admit(s, tts._auto_latent(None), toks[s % N] + [0], torch.rand(400, device="cuda"))
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    steps = 100
    ws.advance(5)
    ev[0].record()
    ws.advance(steps)
    ev[1].record()
    ev[1].synchronize()
    res["pool_step_ms"] = ev[0].elapsed_time(ev[1]) / steps
    ar = tts.autoregressive
    us = [torch.rand(1, 300, device="cuda") for _ in range(C)]
    for _ in range(2):                      # the second call replays the graph the first one captured
        pe = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        ar.generate_grouped([tts._auto_latent(None)] * C, [t + [0] for t in (toks * C)[:C]], [1] * C, 300,
                            uniforms_list=us, stop_check_every=1000, prefill_events=pe)
        ev[1].record()
        ev[1].synchronize()
    res["batch_step_ms"] = (ev[0].elapsed_time(ev[1]) - pe[0].elapsed_time(pe[1])) / 299
    # one admission's prefill, which holds the running streams for its duration
    for s in range(C):
        ws.release(s)
    pre = []
    for s in range(min(C, 8)):
        ev[0].record()
        ws.admit(s, tts._auto_latent(None), toks[s % N] + [0], torch.rand(400, device="cuda"))
        ev[1].record()
        ev[1].synchronize()
        pre.append(ev[0].elapsed_time(ev[1]))
    res["admission_ms_min_max"] = [min(pre), max(pre)]
    pool.close()
    res["gpu_after"] = gpu_state()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
