"""Times the tortoise-detect classifier (`classify_audio_clip`) on one GPU: the engine forward (synthetic weights) at
n = 220 000 samples (the crop is_this_from_tortoise.py applies) and 480 000 (20 s), with CUDA events after warm-up, over
at least a second of calls; one line per level, one for the input conv and one for final + attention + head. As the bar
to beat, the reference AudioMiniEncoderWithClassifierHead (from oracle/_ref) in eager PyTorch fp32, TF32 off, on the
same GPU. Prints the GPU's name, power limit and SM clock, and the engine-vs-reference difference of the logits at
each timed size; the last line is one JSON object."""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _gpu():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def _calls_for(fn, seconds=1.0):
    """Number of calls that fill at least `seconds`, from one timed call after warm-up."""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    fn()
    ev[1].record()
    torch.cuda.synchronize()
    return max(3, int(seconds * 1000.0 / max(ev[0].elapsed_time(ev[1]), 1e-3)) + 1)


def time_engine(eng, wav, seconds=1.0):
    """-> (ms per forward, {stage: ms per forward}) over >= `seconds` of back-to-back forwards."""
    from tortoise_tts_b200.classifier_engine import DEPTH
    ws = eng.workspace(wav.numel())
    stages = ["input conv"] + ["level %d (C=%d, L=%d)" % (l, 32 << l, ws.lens[l]) for l in range(DEPTH)] + \
        ["final + attention + head (T=%d)" % ws.lens[DEPTH]]
    fns = [lambda: eng.front(ws, wav)] + [lambda l=l: eng.level(ws, l) for l in range(DEPTH)] + [lambda: eng.tail(ws)]

    def once(ev=None):
        for i, f in enumerate(fns):
            if ev is not None:
                ev[i].record()
            f()
        if ev is not None:
            ev[-1].record()
    for _ in range(3):
        once()
    reps = _calls_for(once, seconds)
    evs = [[torch.cuda.Event(enable_timing=True) for _ in range(len(fns) + 1)] for _ in range(reps)]
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for ev in evs:
        once(ev)
    t1.record()
    torch.cuda.synchronize()
    per = {s: sum(ev[i].elapsed_time(ev[i + 1]) for ev in evs) / reps for i, s in enumerate(stages)}
    return t0.elapsed_time(t1) / reps, per, reps


def time_reference(model, x, seconds=1.0):
    with torch.no_grad():
        for _ in range(3):
            model(x)
        reps = _calls_for(lambda: model(x), seconds)
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(reps):
            model(x)
        t1.record()
        torch.cuda.synchronize()
    return t0.elapsed_time(t1) / reps, reps


def main():
    import __graft_entry__
    __graft_entry__.build()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    from oracle.ref_shims import load_reference
    from test_classifier_host import make_clip
    from tortoise_tts_b200.classifier_engine import ClassifierEngine
    from tortoise_tts_b200.synth import synth_classifier
    load_reference()
    from tortoise.models.classifier import AudioMiniEncoderWithClassifierHead
    sd = synth_classifier(0)
    eng = ClassifierEngine(sd, device="cuda")
    ref = AudioMiniEncoderWithClassifierHead(2, spec_dim=1, embedding_dim=512, depth=5, downsample_factor=4,
                                             resnet_blocks=2, attn_blocks=4, num_attn_heads=4, base_channels=32,
                                             dropout=0, kernel_size=5, distribute_zero_label=False)
    ref.load_state_dict(sd, strict=True)
    ref = ref.cuda().eval()
    gpu = _gpu()
    print("GPU: %s (name, power limit, SM clock, max SM clock)" % gpu)
    result = {"gpu": gpu, "sizes": {}}
    for n in (220000, 480000):
        clip = make_clip(n).cuda()
        logits, _ = eng.forward(clip)
        with torch.no_grad():
            want = ref(clip.unsqueeze(0))
        diff = (logits - want).abs().max().item()
        ms, per, reps = time_engine(eng, clip.reshape(-1).contiguous())
        ref_ms, ref_reps = time_reference(ref, clip.unsqueeze(0))
        print("n = %d: engine %.3f ms/call (%d calls), reference fp32 eager %.3f ms/call (%d calls), speed-up %.2fx; "
              "max |logit diff| %.2e (logits %s)" % (n, ms, reps, ref_ms, ref_reps, ref_ms / ms, diff,
                                                     [round(v, 4) for v in want[0].tolist()]))
        for s, v in per.items():
            print("    %-34s %8.3f ms  %5.1f %%" % (s, v, 100.0 * v / sum(per.values())))
        result["sizes"][n] = dict(engine_ms=ms, reference_ms=ref_ms, speedup=ref_ms / ms, max_logit_diff=diff,
                                  stages_ms=per)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
