#!/usr/bin/env python
"""Times the phases of the one-kernel decode step (csrc/ar_step.cu) in isolation: for every phase bit, one launch that
runs ONLY that phase for all 30 layers (30 x (phase + grid barrier)), CUDA events, L2 flushed between launches.
Development aid; prints a table.   python tools/ar_step_probe.py [B] [step]"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402


def main():
    from test_gpu_ar_step import _mk
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 256
    step = int(sys.argv[2]) if len(sys.argv) > 2 else 215
    D, H, L, V, P, Nmax = 1024, 16, 30, 8194, 174, 430
    hd, t = _mk(B, D, H, L, V, P, Nmax, step, seed=1)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")

    def timeit(mask, reps=5):
        for _ in range(2):
            hd.step(phase_mask=mask, layer_begin=0, layer_end=L)
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            hd.step(phase_mask=mask, layer_begin=0, layer_end=L)
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ts.sort()
        return ts[len(ts) // 2] * 1e3
    names = ["embed+ln1", "c_attn", "attention", "c_proj", "ln_2", "c_fc", "mlp.c_proj", "ln_1'", "mel_head"]
    print("B=%d step=%d" % (B, step))
    tot = 0.0
    for i, n in enumerate(names):
        us = timeit(1 << i)
        per = us / (L if 0 < i < 8 else 1)
        if 0 < i < 8:
            tot += us
        print("  %-12s %9.1f us total  %7.2f us per layer-phase" % (n, us, per))
    print("  sum of layer phases: %.1f us" % tot)
    print("  whole step:          %.1f us" % timeit(0x1ff))
    print("  two cheap phases (ln_2 + ln_1', 60 barriers): %.1f us" % timeit(16 | 128))
    nop = timeit(512)
    print("  30 empty grid barriers: %.1f us  (%.2f us each incl. launch share)" % (nop, nop / 30))
    assert int(t["state"][2].item()) == 0


if __name__ == "__main__":
    main()
