#!/usr/bin/env python
"""Times the wgmma GEMM variants (tile width, one-tile-per-CTA vs persistent, the warp-specialised 128x256 kernel, cluster
multicast, split-K) on the shapes of the hot path, next to torch.matmul (cuBLAS) as a calibration of what the hardware
delivers on that shape. Development aid; prints a table. L2 is flushed between timed launches."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def timeit(fn, flush, reps=15):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2] * 1e3     # median, us


def main():
    from tortoise_tts_b200 import lib
    dev = "cuda"
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    shapes = [  # name, M, N, K, taps, batch, residual, out
        ("diff conv1x1", 1872, 1024, 1024, 1, 2, True, "f32"),
        ("diff conv k3", 1872, 1024, 1024, 3, 2, True, "f32"),
        ("diff qkv", 1872, 3072, 1024, 1, 2, False, "bf16"),
        ("clvp qkv", 27520, 2304, 768, 1, 1, False, "bf16"),
        ("ar qkv", 256, 3072, 1024, 1, 1, False, "bf16"),
        ("ar fc", 256, 4096, 1024, 1, 1, False, "bf16"),
        ("ar proj2", 256, 1024, 4096, 1, 1, False, "f32"),
    ]
    only = os.environ.get("TTB_SWEEP_SHAPES")            # e.g. "diff": shapes whose name contains the string
    quick = os.environ.get("TTB_SWEEP_QUICK") == "1"      # tile 64 / 128 variants only; adds M = 1920 (no ragged edge)
    if quick:
        shapes += [("diff conv k3 M=1920", 1920, 1024, 1024, 3, 2, True, "f32"),
                   ("diff conv1x1 M=1920", 1920, 1024, 1024, 1, 2, True, "f32")]
    for name, M, N, K, taps, batch, res, out in shapes:
        if only and only not in name:
            continue
        A = torch.randn(batch, M, K, device=dev).to(torch.bfloat16)
        W = (torch.randn(N, taps * K, device=dev) * 0.02).to(torch.bfloat16)
        bias = torch.zeros(N, device=dev)
        of = torch.zeros(batch, M, N, device=dev) if out == "f32" else None
        ob = torch.zeros(batch, M, N, device=dev, dtype=torch.bfloat16) if out == "bf16" else None
        flops = 2.0 * batch * M * N * K * taps
        # cuBLAS calibration: same FLOPs as one [batch*M, taps*K] x [taps*K, N] product, bf16 out
        A2 = torch.randn(batch * M, taps * K, device=dev).to(torch.bfloat16)
        Wt = W.t().contiguous()
        t_cublas = timeit(lambda: torch.matmul(A2, Wt), flush)
        print("== %-13s M=%dx%d N=%d K=%d taps=%d  (%.1f GFLOP)   cuBLAS bf16: %7.1f us  %6.0f TF/s" %
              (name, batch, M, N, K, taps, flops / 1e9, t_cublas, flops / t_cublas / 1e6))
        variants = []
        for tile in ((64, 128) if quick else (32, 64, 128, 256)):
            if M <= 256 and tile == 256:
                continue
            for variant in (1, 2):
                if tile == 256 and variant == 2:
                    continue
                variants.append(dict(tile_n=tile, variant=variant))
            for cl in (2, 4):
                if tile != 256 and ((N + tile - 1) // tile) % cl == 0:
                    variants.append(dict(tile_n=tile, cluster=cl))
        if M > 256:
            variants.append(dict(variant=7))                   # persistent warp-specialised 128x256 (gemm_ws.cuh)
        if os.environ.get("TTB_TEST_EXPERIMENTAL") == "1" and M > 256:
            variants += [dict(tile_n=128, variant=5)]          # two TMA issuer threads
        if name == "ar proj2":
            variants = [dict(tile_n=t, splitk=s, cluster=c) for t in (32, 64, 128) for s in (2, 4, 8) for c in (0, 4)
                        if c == 0 or ((N + t - 1) // t) % c == 0]
        for v in variants:
            kw = dict(M=M, N=N, K=K, taps=taps, pad=(taps - 1) // 2, batch=batch, a_bstride=M * K)
            sk = v.get("splitk", 1)
            if sk > 1:
                part = torch.zeros(sk, M, N, device=dev)
                fn = lambda: lib.gemm(A, W, out_f32=part, outf_bstride=M * N, **kw, **v)
            else:
                fn = lambda: lib.gemm(A, W, bias=bias, residual=of if res else None, out_f32=of, out_bf16=ob,
                                      res_bstride=M * N, outf_bstride=M * N, outb_bstride=M * N, **kw, **v)
            try:
                t = timeit(fn, flush)
                print("   %-48s %7.1f us  %6.0f TF/s" % (str(v), t, flops / t / 1e6))
            except Exception as e:  # noqa: BLE001
                print("   %-48s failed: %s" % (str(v), str(e)[:80]))


if __name__ == "__main__":
    main()
