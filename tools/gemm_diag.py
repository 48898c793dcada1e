#!/usr/bin/env python
"""Where does the wgmma GEMM spend its time?
 (1) per-launch time of back-to-back launches (host latency amortised, warm L2) next to torch.matmul (cuBLAS);
 (2) per-CTA phase timestamps (ttb_debug_gemm_trace): setup, first operand latency, mainloop, drain, epilogue, and
     how many CTAs an SM really runs at a time.
Development aid."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def per_launch_us(fn, n=20, reps=7):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) / n)
    ts.sort()
    return ts[len(ts) // 2] * 1e3


def trace(lib, fn, ctas, label):
    buf = torch.zeros(ctas * 8, dtype=torch.int64, device="cuda")
    fn()
    torch.cuda.synchronize()
    lib.debug_gemm_trace(buf)
    fn()
    torch.cuda.synchronize()
    lib.debug_gemm_trace(None)
    t = buf.view(ctas, 8).cpu().double()
    t0 = t[:, 0].min()
    span = (t[:, 7].max() - t0).item()
    ph = {
        "setup (barriers, dependency wait)": t[:, 2] - t[:, 0],
        "consumers reach the main loop": t[:, 3] - t[:, 2],
        "main loop (wgmma retired)": t[:, 4] - t[:, 3],
        "accumulator staged": t[:, 5] - t[:, 4],
        "epilogue": t[:, 6] - t[:, 5],
        "tail": t[:, 7] - t[:, 6],
        "CTA lifetime": t[:, 7] - t[:, 0],
    }
    print("-- trace %s: %d CTAs, kernel span %.1f us, sum(lifetime)/(span*SMs) = %.2f CTAs resident per SM on average"
          % (label, ctas, span / 1e3, (ph["CTA lifetime"].sum().item() / (span * torch.cuda.get_device_properties(0).multi_processor_count))))
    for k, v in ph.items():
        print("   %-26s mean %7.2f us   p10 %7.2f   p90 %7.2f" % (k, v.mean().item() / 1e3, v.quantile(0.1).item() / 1e3,
                                                                    v.quantile(0.9).item() / 1e3))
    sm = t[:, 1].long()
    for s in (0, 77):
        idx = (sm == s).nonzero().flatten()
        rows = sorted([(t[i, 0].item() - t0.item(), t[i, 3].item() - t0.item(), t[i, 5].item() - t0.item(),
                        t[i, 7].item() - t0.item()) for i in idx])[:8]
        print("   SM %d timeline (us) [start, first-mma, accum-ready, end]: " % s +
              "  ".join("[%.1f %.1f %.1f %.1f]" % tuple(x / 1e3 for x in r) for r in rows))


def main():
    from tortoise_tts_b200 import lib
    dev = "cuda"
    shapes = [  # name, M, N, K, taps, batch, residual, out
        ("diff conv1x1", 1872, 1024, 1024, 1, 2, True, "f32"),
        ("diff conv k3", 1872, 1024, 1024, 3, 2, True, "f32"),
        ("diff qkv", 1872, 3072, 1024, 1, 2, False, "bf16"),
        ("clvp qkv", 27520, 2304, 768, 1, 1, False, "bf16"),
        ("ar qkv", 256, 3072, 1024, 1, 1, False, "bf16"),
        ("ar fc", 256, 4096, 1024, 1, 1, False, "bf16"),
        ("ar proj", 256, 1024, 1024, 1, 1, False, "bf16"),
    ]
    only = sys.argv[1] if len(sys.argv) > 1 else ""
    for name, M, N, K, taps, batch, res, out in shapes:
        if only and not name.startswith(only):
            continue
        A = torch.randn(batch, M, K, device=dev).to(torch.bfloat16)
        W = (torch.randn(N, taps * K, device=dev) * 0.02).to(torch.bfloat16)
        bias = torch.zeros(N, device=dev)
        of = torch.zeros(batch, M, N, device=dev) if out == "f32" else None
        ob = torch.zeros(batch, M, N, device=dev, dtype=torch.bfloat16) if out == "bf16" else None
        flops = 2.0 * batch * M * N * K * taps
        A2 = torch.randn(batch * M, taps * K, device=dev).to(torch.bfloat16)
        Wt = W.t().contiguous()
        o2 = torch.empty(batch * M, N, device=dev, dtype=torch.bfloat16)
        tc = per_launch_us(lambda: torch.matmul(A2, Wt, out=o2))
        print("== %-13s %dx%d N=%d K=%d taps=%d (%.1f GFLOP)  cuBLAS %.1f us = %.0f TF/s" %
              (name, batch, M, N, K, taps, flops / 1e9, tc, flops / tc / 1e6))
        kw = dict(M=M, N=N, K=K, taps=taps, pad=(taps - 1) // 2, batch=batch, a_bstride=M * K, res_bstride=M * N,
                  outf_bstride=M * N, outb_bstride=M * N)
        tiles = [32] if M <= 256 else [64, 128]
        if M <= 256:          # one-tile kernel, 5 stages (variant 3) against 4 stages (variant 4)
            for v, nm in ((3, "5 stages"), (4, "4 stages")):
                t1 = per_launch_us(lambda: lib.gemm(A, W, bias=bias, out_bf16=ob, tile_n=32, variant=v, **kw))
                print("   tile  32 one-tile %s: %.1f us" % (nm, t1))
            for v, nm in ((3, "8 stages, 1 CTA/SM"), (1, "4 stages")):
                t1 = per_launch_us(lambda: lib.gemm(A, W, bias=bias, out_bf16=ob, tile_n=64, variant=v, **kw))
                print("   tile  64 one-tile %s: %.1f us" % (nm, t1))
                trace(lib, lambda: lib.gemm(A, W, bias=bias, out_bf16=ob, tile_n=64, variant=v, **kw),
                      ((N + 63) // 64) * ((M + 127) // 128) * batch, "%s tile 64 %s" % (name, nm))
        for tile in tiles:
            for variant in (1, 2):
                full = lambda: lib.gemm(A, W, bias=bias, residual=of if res else None, out_f32=of, out_bf16=ob,
                                        tile_n=tile, variant=variant, **kw)
                bare = lambda: lib.gemm(A, W, tile_n=tile, variant=variant, **kw)
                t1, t2 = per_launch_us(full), per_launch_us(bare)
                print("   tile %3d %-10s full epilogue %7.1f us = %5.0f TF/s     no output %7.1f us" %
                      (tile, "one-tile" if variant == 1 else "persistent", t1, flops / t1 / 1e6, t2))
            if tile == tiles[-1]:
                ctas = ((N + tile - 1) // tile) * ((M + 127) // 128) * batch
                trace(lib, lambda: lib.gemm(A, W, bias=bias, residual=of if res else None, out_f32=of, out_bf16=ob,
                                            tile_n=tile, variant=1, **kw), ctas, "%s tile %d" % (name, tile))


if __name__ == "__main__":
    main()
