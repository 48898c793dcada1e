"""tts_batch against a tts_with_preset loop on one GPU, with CUDA events.

Workload: the 8 utterances of bench.py's config5 (the para53 paragraph cycled to 169 ... 337 BPE tokens), full-size
synthetic checkpoint with the stop token suppressed (every candidate decodes all 430 mel tokens), presets 'ultra_fast'
(16 candidates per utterance) and 'fast' (96). The two arms run alternately, three times each, in one process, with
the same seed and conditioning. Reports per preset and arm the AR-stage and total device ms (CUDA events), audio-s/s,
the token agreement of the decoded candidates and the largest waveform difference between the arms, and the card's
name, power limit and SM clock read in the same run. Needs a CUDA device (there is no CPU fallback)."""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _gpu():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def main():
    import __graft_entry__ as ge
    ge.build()
    import bench
    from tortoise_tts_b200.api import TextToSpeech
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_all
    cfg = ModelConfig.full()
    tts = TextToSpeech(state_dicts=synth_all(cfg, seed=0, suppress_stop=True), config=cfg, kv_cache=True)
    utt = bench.config5_tokens(bench.load_tokens())
    g = torch.Generator().manual_seed(0)
    cond = (torch.randn(1, cfg.ar_dim, generator=g) * 0.5, torch.randn(1, 2 * cfg.diff_dim, generator=g) * 0.3)
    kw = dict(conditioning_latents=cond, max_mel_tokens=430, verbose=False, use_deterministic_seed=1234)
    ar = tts.autoregressive
    codes = []                                   # the decoded candidates of the current run, in utterance order
    gen, gen_grouped = ar.generate, ar.generate_grouped
    ar.generate = lambda *a, **k: codes.append(gen(*a, **k)) or codes[-1]
    ar.generate_grouped = lambda *a, **k: codes.extend(gen_grouped(*a, **k)) or codes[-len(a[2]):]

    def run(arm, preset):
        codes.clear()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        torch.cuda.synchronize()
        ev[0].record()
        if arm == "loop":
            wavs, ar_ms = [], 0.0
            for u, t in enumerate(utt):
                wavs.append(tts.tts_with_preset("u%d" % u, preset=preset, text_tokens=t, **kw))
                ar_ms += tts.last_timings["ar_ms"]
        else:
            wavs = tts.tts_batch(["u%d" % u for u in range(len(utt))], preset=preset, text_tokens_list=utt, **kw)
            ar_ms = tts.last_timings["ar_ms"]
        ev[1].record()
        torch.cuda.synchronize()
        total = ev[0].elapsed_time(ev[1])
        audio_s = sum(w.shape[-1] for w in wavs) / 24000.0
        return dict(ar_ms=ar_ms, total_ms=total, audio_s_per_s=audio_s / (total / 1e3)), wavs, [c.cpu() for c in codes]

    res = {"gpu": _gpu(), "workload": "config5 utterances (%s tokens), 430 mel tokens, stop token suppressed, k=1"
           % "/".join(str(len(u)) for u in utt), "presets": {}}
    for preset in ("ultra_fast", "fast"):
        for arm in ("loop", "batch"):             # warm-up: module loading, graph capture of every decode shape
            run(arm, preset)
        runs = {"loop": [], "batch": []}
        outs = {}
        for _ in range(3):
            for arm in ("loop", "batch"):
                r, wavs, cs = run(arm, preset)
                runs[arm].append(r)
                outs[arm] = (wavs, cs)
        agree = torch.cat([(a == b).float().reshape(-1) for a, b in zip(outs["loop"][1], outs["batch"][1])]).mean().item()
        dw = max((a.reshape(-1)[: min(a.numel(), b.numel())] - b.reshape(-1)[: min(a.numel(), b.numel())]).abs().max().item()
                 for a, b in zip(outs["loop"][0], outs["batch"][0]))
        res["presets"][preset] = {arm: {k: [round(r[k], 2) for r in rs] for k in rs[0]} for arm, rs in runs.items()}
        res["presets"][preset]["token_agreement"] = agree
        res["presets"][preset]["max_abs_dwav"] = dw
        res["presets"][preset]["decode_mode"] = "%s, %d chain(s)" % (ar._dec["mode"], len(ar._dec["chains"]))
        print(json.dumps({preset: res["presets"][preset]}), flush=True)
    res["gpu_after"] = _gpu()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
