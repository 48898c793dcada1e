"""Times the `api_fast` path (SURVEY 8f row 3) at full size on one H100: `tts()` (one sequence -> latents -> HiFiGAN)
and `tts_stream()` (first-chunk latency, total). Synthetic checkpoint with the stop token suppressed, so `tts()` runs
the model's 603-token limit and the stream runs `500 - prompt` tokens (autoregressive.py:553,571). Prints one JSON line.
The reference publishes, for this path only, "RTF 0.25-0.3" and "< 500 ms" to the first chunk on an unnamed GPU
(README.md:34; BASELINE.md §1) — quoted next to the numbers, not a like-for-like baseline."""
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from tortoise_tts_b200 import api_fast
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_autoregressive, synth_hifigan, synth_rlg
    cfg = ModelConfig.full()
    sds = {"autoregressive": synth_autoregressive(cfg, 0, True), "hifigan": synth_hifigan(cfg, 0),
           "rlg_auto": synth_rlg(cfg.ar_dim, 0)}
    with open(os.path.join(ROOT, "tests", "golden", "bench_text_tokens.json")) as f:
        toks = json.load(f)["para53"]["tokens"]
    tts = api_fast.TextToSpeech(state_dicts=sds, config=cfg, kv_cache=True)
    res = {"path": "api_fast (one AR sequence -> GPT latents -> HiFiGAN)", "text_tokens": len(toks)}
    for it in range(3):                                   # the last of three runs is reported (graphs captured, caches warm)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        wav = tts.tts("unused", text_tokens=toks, use_deterministic_seed=1, verbose=False)
        wav_host = wav.cpu()
        t1 = time.perf_counter()
        res["tts"] = {"wall_ms": (t1 - t0) * 1e3, "audio_s": wav_host.shape[-1] / 24000.0,
                      "audio_s_per_s": wav_host.shape[-1] / 24000.0 / (t1 - t0), **tts.last_timings}
    for it in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        first = None
        n = 0
        for chunk in tts.tts_stream("unused", text_tokens=toks, use_deterministic_seed=1, verbose=False):
            c = chunk.cpu()
            n += c.numel()
            if first is None:
                first = time.perf_counter() - t0
        t1 = time.perf_counter()
        res["tts_stream"] = {"first_chunk_ms": first * 1e3, "wall_ms": (t1 - t0) * 1e3, "audio_s": n / 24000.0,
                             "audio_s_per_s": n / 24000.0 / (t1 - t0), "stream_chunk_size": 40}
    res["reference_published"] = "README.md:34: RTF 0.25-0.3 (3.3-4 audio-s/s), first chunk < 500 ms, GPU unnamed"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
