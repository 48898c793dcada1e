"""Times prompt redaction on one GPU: the wav2vec2-large-robust aligner forward (synthetic weights, full size) plus the
host alignment and cut, on a 20 s clip at 24 kHz, with CUDA events; and the same model as HF Wav2Vec2ForCTC in fp32
eager PyTorch on the same GPU. Prints one JSON line with the GPU's name and power limit."""
import json
import math
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _gpu():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def _time(fn, reps):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    out = []
    for _ in range(reps):
        ev[0].record()
        fn()
        ev[1].record()
        torch.cuda.synchronize()
        out.append(ev[0].elapsed_time(ev[1]))
    out.sort()
    return {"median_ms": out[len(out) // 2], "min_ms": out[0]}


def main(seconds=20.0, reps=20):
    import torchaudio
    from transformers import Wav2Vec2Config, Wav2Vec2ForCTC
    from tortoise_tts_b200 import redaction
    from tortoise_tts_b200.synth import synth_wav2vec
    from tortoise_tts_b200.wav2vec_engine import Wav2VecEngine
    cfg, sd, vocab = synth_wav2vec("full", seed=0)
    eng = Wav2VecEngine(cfg, sd, "cuda")
    tok = redaction.CTCCharTokenizer(vocab)
    aligner = redaction.Aligner(eng, tok)
    n = int(seconds * 24000)
    t = torch.arange(n) / 24000.0
    wav = (0.1 * torch.sin(2 * math.pi * 220 * t) + 0.02 * torch.randn(n, generator=torch.Generator().manual_seed(0)))
    wav = wav.reshape(1, -1).cuda()
    text = "[I am really sad,] please feed me. " * 4
    T = eng._workspace(n).T
    H, C, FF, L = eng.H, eng.C, eng.FF, eng.L
    lens = eng._workspace(n).lens
    flop = 2 * lens[0] * C * 10 + sum(2 * lens[i] * C * C * (3 if i < 5 else 2) for i in range(1, 7))
    flop += 2 * T * C * H + 2 * T * H * (H // eng.groups) * eng.pos_k
    flop += L * (2 * T * H * 4 * H + 4 * T * T * H + 4 * T * H * FF) + 2 * T * H * eng.V
    for _ in range(3):
        eng.logits(wav)
    torch.cuda.synchronize()
    res = {"gpu": _gpu(), "clip_s": seconds, "frames": T, "model_gflop": flop / 1e9}
    res["aligner_forward"] = _time(lambda: eng.ids(wav), reps)
    res["aligner_forward"]["tflops"] = flop / (res["aligner_forward"]["median_ms"] * 1e-3) / 1e12
    walls = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        aligner.redact(wav, text)
        torch.cuda.synchronize()
        walls.append((time.perf_counter() - t0) * 1e3)
    walls.sort()
    res["redact_wall_ms"] = {"median_ms": walls[len(walls) // 2], "min_ms": walls[0]}
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    m = Wav2Vec2ForCTC(Wav2Vec2Config(**cfg)).eval()
    m.load_state_dict(sd)
    m = m.cuda()

    def hf():
        with torch.no_grad():
            a = torchaudio.functional.resample(wav, 24000, 16000)
            m((a - a.mean()) / torch.sqrt(a.var() + 1e-7)).logits.argmax(-1)
    for _ in range(3):
        hf()
    res["hf_fp32_eager_forward"] = _time(hf, reps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
