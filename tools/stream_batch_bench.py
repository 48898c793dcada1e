"""Times api_fast.TextToSpeech.tts_stream_batch (R listeners served by one decode batch) against a loop of tts_stream
calls (how R listeners are served one after the other), on the full-size synthetic checkpoint with the stop token
suppressed (every stream decodes to its cap, 500 - prompt positions). Seeded token lists of 40-90 tokens. Rounds
alternate the arms. Every stream's chunk arrival times come from a host clock read after a device synchronise at each
chunk; the loop arm serves listener u after listeners 0 .. u-1 have finished, and a loop over more streams than
--loop-streams is not run (its rows are reported as not measured).

Per R: time to the first chunk of the slowest listener, wall time, audio seconds per second, and playback underruns. A
listener starts playing at its first chunk; an underrun is a later chunk that arrives after the audio before it has
finished playing (24 kHz). Also: the largest R without an underrun, and the GPU's name, power limit and SM clock, read
in the same run. Prints one JSON line.

    python tools/stream_batch_bench.py [--sizes 1 8 32 64 128 256] [--rounds 3] [--loop-streams 8]
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

SR = 24000.0


def listener_stats(arrivals):
    """arrivals: [(t_seconds, samples), ...] of one listener in order -> (first chunk time, underruns, audio seconds)."""
    t0 = arrivals[0][0]
    played_until, under = t0, 0
    for t, n in arrivals:
        if t > played_until + 1e-9 and t != t0:
            under += 1
        played_until = max(played_until, t) + n / SR
    return t0, under, sum(n for _, n in arrivals) / SR


def summarize(per_listener, wall):
    firsts, unders, audio = zip(*[listener_stats(a) for a in per_listener])
    return {"first_chunk_worst_ms": max(firsts) * 1e3, "wall_ms": wall * 1e3, "audio_s": sum(audio),
            "audio_s_per_s": sum(audio) / wall, "underruns": sum(unders),
            "listeners_with_underrun": sum(1 for x in unders if x)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[1, 8, 32, 64, 128, 256])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--loop-streams", type=int, default=8, help="largest R the tts_stream loop arm runs")
    ap.add_argument("--chunk", type=int, default=40, help="stream_chunk_size")
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("stream_batch_bench needs a CUDA device")
    from tortoise_tts_b200 import api_fast
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_autoregressive, synth_hifigan, synth_rlg
    cfg = ModelConfig()
    sds = {"autoregressive": synth_autoregressive(cfg, 0, True), "hifigan": synth_hifigan(cfg, 0),
           "rlg_auto": synth_rlg(cfg.ar_dim, 0)}
    tts = api_fast.TextToSpeech(state_dicts=sds, config=cfg, kv_cache=True)
    n_all = max(args.sizes)
    g = torch.Generator().manual_seed(args.seed)
    lens = torch.randint(40, 91, (n_all,), generator=g).tolist()
    toks = [torch.randint(1, 255, (n,), generator=g).tolist() for n in lens]
    kw = dict(use_deterministic_seed=1, verbose=False, stream_chunk_size=args.chunk)
    res = {"gpu_before": gpu_state(), "text_tokens": [min(lens), max(lens)], "sizes": args.sizes,
           "rounds": args.rounds, "stream_chunk_size": args.chunk, "loop_streams": args.loop_streams}

    def run_batch(n):
        arr = [[] for _ in range(n)]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for u, chunk, last in tts.tts_stream_batch(["x"] * n, text_tokens_list=toks[:n], **kw):
            torch.cuda.synchronize()
            arr[u].append((time.perf_counter() - t0, int(chunk.numel())))
        wall = time.perf_counter() - t0
        tim = {k: v for k, v in tts.last_timings.items() if k.endswith("_ms")}
        return {**summarize(arr, wall), **tim}, [sum(c for _, c in a) for a in arr]

    def run_loop(n):
        arr = [[] for _ in range(n)]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for u in range(n):
            for chunk in tts.tts_stream("x", text_tokens=toks[u], **kw):
                torch.cuda.synchronize()
                arr[u].append((time.perf_counter() - t0, int(chunk.numel())))
        wall = time.perf_counter() - t0
        return summarize(arr, wall), [sum(c for _, c in a) for a in arr]

    # warm-up: modules, the one-row step graph and every batch size's workspace and graph
    list(tts.tts_stream("x", text_tokens=toks[0], **kw))
    for n in args.sizes:
        run_batch(n)
    rounds = []
    for r in range(args.rounds):
        rd = {"loop": {}, "batch": {}}
        for n in args.sizes:
            if n <= args.loop_streams:
                rd["loop"][n], llen = run_loop(n)
            rd["batch"][n], blen = run_batch(n)
            if n in rd["loop"]:
                assert blen == llen, "stream lengths differ between the arms"
        rounds.append(rd)
    res["rounds_data"] = rounds
    summ, clean = {}, []
    for n in args.sizes:
        for arm in ("loop", "batch"):
            if n not in rounds[0][arm]:
                summ["%s_%d" % (arm, n)] = "not measured"
                continue
            keys = rounds[0][arm][n].keys()
            summ["%s_%d" % (arm, n)] = {k: [round(min(rd[arm][n][k] for rd in rounds), 1),
                                            round(max(rd[arm][n][k] for rd in rounds), 1)] for k in keys}
        if all(rd["batch"][n]["underruns"] == 0 for rd in rounds):
            clean.append(n)
    res["summary_min_max"] = summ
    res["largest_R_without_underrun"] = max(clean) if clean else 0
    res["gpu_after"] = gpu_state()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
