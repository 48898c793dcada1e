import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from tortoise_tts_b200.config import ModelConfig
from tortoise_tts_b200.synth import synth_all
from tortoise_tts_b200 import ar_engine
cfg = ModelConfig.medium()
sd = synth_all(cfg, seed=1, suppress_stop=True)["autoregressive"]
torch.manual_seed(0)
text = torch.randint(1, 255, (169,)).tolist() + [0]
cond = torch.randn(1, cfg.ar_dim)
default_mode = ar_engine.AREngine.MODE
for B in (256, 32, 3):
    N = 20
    u = torch.rand(B, N)
    runs = {}
    for fused in (1, 0, 1):
        ar_engine.AREngine.MODE = default_mode if fused else "perop"
        eng = ar_engine.AREngine(sd, cfg)
        tr = []
        codes = eng.generate(cond, text, B, N, uniforms=u, trace_logits=tr).cpu()
        key = fused if fused not in runs else 2
        runs[key] = (codes, torch.stack([x.cpu() for x in tr], 1))
        del eng
    c1, l1 = runs[1]; c0, l0 = runs[0]; c2, l2 = runs[2]
    print("B", B, "fused run1 == fused run2:", torch.equal(c1, c2), "logits equal:", torch.equal(l1, l2))
    first = []
    for b in range(B):
        same = (c1[b] == c0[b]).long().cumprod(0)
        first.append(int(same.sum()))
    ft = torch.tensor(first)
    print(" first-divergence histogram:", torch.bincount(ft, minlength=N + 1).tolist())
    per_pos = [(l1[:, i] - l0[:, i]).abs().max().item() for i in range(N)]
    print(" max |dlogit| per position (all rows):", ["%.2e" % v for v in per_pos])
    print(" logit scale:", l0.abs().max().item(), " std:", l0.std().item())
    # a diverging row
    for b in range(B):
        p = first[b]
        if p < N:
            d = (l1[b, p] - l0[b, p]).abs().max().item()
            top1 = torch.topk(l1[b, p], 5); top0 = torch.topk(l0[b, p], 5)
            print(" row", b, "diverges at", p, "tokens", int(c1[b, p]), int(c0[b, p]), "max dlogit there %.3e" % d)
            print("   top5 fused ", top1.values.tolist(), top1.indices.tolist())
            print("   top5 per-op", top0.values.tolist(), top0.indices.tolist())
            srt = torch.sort(l0[b, p], descending=True).values
            print("   gaps around rank 50:", (srt[45:55][:-1] - srt[45:55][1:]).tolist())
            break
