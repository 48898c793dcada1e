"""tortoise-detect classifier on the sm_90a kernels: the AudioMiniEncoderWithClassifierHead forward that
`classify_audio_clip` runs (tortoise/api.py:133-145, models/classifier.py).

    waveform [n] -> init Conv1d(1, 32, k3)                              fp32 ttb_voc_conv1d + ttb_transpose_f32
      -> 5 levels, C = 32 * 2^l: 2 x ResBlock (GN -> SiLU -> conv5, twice; identity skip), then Downsample
         Conv1d(C, 2C, k5, stride 4, p2)                               ttb_groupnorm + ttb_gemm (taps)
      -> final GN(1024) -> SiLU -> Conv1d(1024, 512, k1)
      -> 4 x AttentionBlock(512, 4 heads of 128)                        ttb_attention(head_dim = 128)
      -> position 0 -> Linear(512, 2)                                   ttb_linear_small

The residual stream is token-major fp32 [L, C]; GEMM operands are bf16. The input conv stays fp32 because the
waveform is the raw input. Level 0 has 32 channels, half the 64-wide K step of ttb_gemm: its GroupNorm writes a bf16
buffer with ldo = 64 whose columns 32-63 stay zero, against weights zero-padded to match. That doubles the MMA work of
the four level-0 convs, which are bound by memory traffic anyway (the fp32 residual stream read and written per conv is
larger than the bf16 operand), and it keeps one GEMM row per sample; the pair view [L/2, 64] instead leaves a
garbage row after an odd L that the Downsample would read and would need clearing.

The Downsample reads a QUAD VIEW of the bf16 copy of the stream: rows [L, C] as [ceil(L/4), 4C], so output row t
(input positions 4t-2 .. 4t+2) is quad rows t-1 (slots 2, 3) and t (slots 0-2): a 2-tap GEMM with pad 1 and K = 4C,
the unused weight slots zero. The buffer is zero past row L. Only checkpoints of this architecture are accepted
(`check_state_dict`).
"""
import math

import torch

from . import lib
from .diffusion_engine import _AttnW, _bf, _f, _groups_for

BASE, DEPTH, RES_BLOCKS, ATTN_BLOCKS, HEADS, EMB, KSIZE, FACTOR = 32, 5, 2, 4, 4, 512, 5, 4


def expected_shapes():
    """Key -> shape of the `classifier.pth` state dict that `classify_audio_clip` builds (122 tensors)."""
    s = {"enc.init.0.weight": (BASE, 1, 3), "enc.init.0.bias": (BASE,)}
    C, i = BASE, 0
    for _ in range(DEPTH):
        for _ in range(RES_BLOCKS):
            p = f"enc.res.{i}."
            for n in ("in_layers.0", "out_layers.0"):
                s[p + n + ".weight"] = s[p + n + ".bias"] = (C,)
            for n in ("in_layers.2", "out_layers.3"):
                s[p + n + ".weight"], s[p + n + ".bias"] = (C, C, KSIZE), (C,)
            i += 1
        s[f"enc.res.{i}.op.weight"], s[f"enc.res.{i}.op.bias"] = (2 * C, C, KSIZE), (2 * C,)
        C, i = 2 * C, i + 1
    s["enc.final.0.weight"] = s["enc.final.0.bias"] = (C,)
    s["enc.final.2.weight"], s["enc.final.2.bias"] = (EMB, C, 1), (EMB,)
    for a in range(ATTN_BLOCKS):
        p = f"enc.attn.{a}."
        s[p + "norm.weight"] = s[p + "norm.bias"] = (EMB,)
        s[p + "qkv.weight"], s[p + "qkv.bias"] = (3 * EMB, EMB, 1), (3 * EMB,)
        s[p + "proj_out.weight"], s[p + "proj_out.bias"] = (EMB, EMB, 1), (EMB,)
    s["head.weight"], s["head.bias"] = (2, EMB), (2,)
    return s


def check_state_dict(sd):
    """Raise ValueError unless `sd` is a classifier.pth of the architecture classify_audio_clip builds."""
    want = expected_shapes()
    bad = []
    missing, extra = sorted(set(want) - set(sd)), sorted(set(sd) - set(want))
    if missing:
        bad.append("missing %s" % ", ".join(missing[:4]) + (" and %d more" % (len(missing) - 4) if len(missing) > 4 else ""))
    if extra:
        bad.append("unexpected %s" % ", ".join(extra[:4]) + (" and %d more" % (len(extra) - 4) if len(extra) > 4 else ""))
    for k in sorted(set(want) & set(sd)):
        if tuple(sd[k].shape) != want[k]:
            bad.append("%s has shape %s, expected %s" % (k, tuple(sd[k].shape), want[k]))
    if bad:
        raise ValueError("unsupported classifier checkpoint (AudioMiniEncoderWithClassifierHead(2, spec_dim=1, "
                         "embedding_dim=512, depth=5, base_channels=32, kernel_size=5) expected): " + "; ".join(bad))


def level_lengths(n):
    """Rows of the residual stream at each level, then after the last Downsample (ceil(L / 4) per level)."""
    lens = [n]
    for _ in range(DEPTH):
        lens.append(-(-lens[-1] // FACTOR))
    return lens


class _Workspace:
    """Every buffer of one forward at one clip length (allocated once per length)."""

    def __init__(self, eng, n):
        dev = eng.dev
        f32, bf = dict(dtype=torch.float32, device=dev), dict(dtype=torch.bfloat16, device=dev)
        self.n = n
        self.lens = lens = level_lengths(n)
        self.y0 = torch.empty(BASE, n, **f32)                           # init conv, channel-major
        self.x, self.h, self.a, self.xb = [], [], [], []
        for l in range(DEPTH):
            L, C = lens[l], BASE << l
            self.x.append(torch.empty(L, C, **f32))                     # residual stream
            self.h.append(torch.empty(L, C, **f32))                     # first conv of a ResBlock
            self.a.append(torch.zeros(L, max(C, 64), **bf))             # GroupNorm output (level 0: columns 32-63 zero)
            self.xb.append(torch.zeros(FACTOR * lens[l + 1], C, **bf))  # bf16 stream for the Downsample, zero past L
        T, Cf = lens[DEPTH], BASE << DEPTH
        self.xf = torch.empty(T, Cf, **f32)
        self.af = torch.empty(T, Cf, **bf)
        self.y = torch.empty(T, EMB, **f32)
        self.ay = torch.empty(T, EMB, **bf)
        self.qkv = torch.empty(T, 3 * EMB, **bf)
        self.o = torch.empty(T, EMB, **bf)
        self.logits = torch.empty(1, 2, **f32)


class ClassifierEngine:
    def __init__(self, sd, device="cuda"):
        check_state_dict(sd)
        self.dev = dev = torch.device(device)
        self.w_init = _f(sd["enc.init.0.weight"], dev)                  # [32, 1, 3] (ttb_voc_conv1d layout)
        self.b_init = _f(sd["enc.init.0.bias"], dev)
        self.levels = []
        C, i = BASE, 0
        for _ in range(DEPTH):
            kc = max(C, 64)
            res = []
            for _ in range(RES_BLOCKS):
                p = f"enc.res.{i}."
                convs = []
                for n in ("in_layers.2", "out_layers.3"):
                    w = torch.zeros(C, KSIZE, kc)
                    w[:, :, :C] = sd[p + n + ".weight"].float().permute(0, 2, 1)      # [out, in, k] -> [out, tap, in]
                    convs.append((_bf(w.reshape(C, KSIZE * kc), dev), _f(sd[p + n + ".bias"], dev)))
                res.append(dict(g1=_f(sd[p + "in_layers.0.weight"], dev), b1=_f(sd[p + "in_layers.0.bias"], dev),
                                g2=_f(sd[p + "out_layers.0.weight"], dev), b2=_f(sd[p + "out_layers.0.bias"], dev),
                                conv1=convs[0], conv2=convs[1]))
                i += 1
            w = sd[f"enc.res.{i}.op.weight"].float()                       # [2C, C, 5]
            wq = torch.zeros(2 * C, 2, FACTOR, C)                           # [out, tap, slot, in] over quad rows t-1, t
            wq[:, 0, 2], wq[:, 0, 3] = w[:, :, 0], w[:, :, 1]
            wq[:, 1, 0], wq[:, 1, 1], wq[:, 1, 2] = w[:, :, 2], w[:, :, 3], w[:, :, 4]
            self.levels.append(dict(C=C, kc=kc, groups=_groups_for(C), res=res,
                                    w_down=_bf(wq.reshape(2 * C, 2 * FACTOR * C), dev),
                                    b_down=_f(sd[f"enc.res.{i}.op.bias"], dev)))
            C, i = 2 * C, i + 1
        self.Cf = C
        self.gf_g, self.gf_b = _f(sd["enc.final.0.weight"], dev), _f(sd["enc.final.0.bias"], dev)
        self.w_final, self.b_final = _bf(sd["enc.final.2.weight"].reshape(EMB, C), dev), _f(sd["enc.final.2.bias"], dev)
        self.attn = [_AttnW(sd, f"enc.attn.{a}.", EMB, HEADS, dev) for a in range(ATTN_BLOCKS)]
        self.w_head, self.b_head = _f(sd["head.weight"], dev), _f(sd["head.bias"], dev)
        self.part = lib.groupnorm_scratch(1, 32, dev)                   # groups <= 32 at every width used here
        self._ws = {}

    def workspace(self, n):
        ws = self._ws.get(n)
        if ws is None:
            if len(self._ws) >= 4:           # a few clip lengths at a time; do not grow without bound
                self._ws.clear()
            ws = self._ws[n] = _Workspace(self, n)
        return ws

    # The forward in stages (tools/classifier_bench.py times each one)
    def front(self, ws, wav):
        """init conv on the fp32 waveform -> level-0 stream fp32 [n, 32]."""
        lib.voc_conv1d(wav, 1, ws.n, self.w_init, self.b_init, BASE, 3, ws.y0)
        lib.transpose_f32(ws.y0, BASE, ws.n, ws.x[0])

    def level(self, ws, l):
        """2 ResBlocks and the Downsample of level l: stream [L, C] -> next stream [ceil(L / 4), 2C]."""
        lv = self.levels[l]
        L, Lq, C, kc, G = ws.lens[l], ws.lens[l + 1], lv["C"], lv["kc"], lv["groups"]
        x, h, a, xb = ws.x[l], ws.h[l], ws.a[l], ws.xb[l]
        for r, rb in enumerate(lv["res"]):
            lib.groupnorm(x, 1, L, C, G, rb["g1"], rb["b1"], self.part, silu=True, out_bf16=a, ldo=kc)
            w, b = rb["conv1"]
            lib.gemm(a, w, M=L, N=C, K=kc, taps=KSIZE, pad=KSIZE // 2, bias=b, out_f32=h, w_static=True)
            lib.groupnorm(h, 1, L, C, G, rb["g2"], rb["b2"], self.part, silu=True, out_bf16=a, ldo=kc)
            w, b = rb["conv2"]
            last = r == RES_BLOCKS - 1
            lib.gemm(a, w, M=L, N=C, K=kc, taps=KSIZE, pad=KSIZE // 2, bias=b, residual=x, out_f32=x,
                     out_bf16=xb if last else None, w_static=True)
        nxt = ws.x[l + 1] if l + 1 < DEPTH else ws.xf
        lib.gemm(xb, lv["w_down"], M=Lq, N=2 * C, K=FACTOR * C, taps=2, pad=1, bias=lv["b_down"], out_f32=nxt,
                 w_static=True)

    def tail(self, ws):
        """final, the 4 AttentionBlocks and the head on position 0 -> logits fp32 [1, 2]."""
        T, Cf = ws.lens[DEPTH], self.Cf
        lib.groupnorm(ws.xf, 1, T, Cf, _groups_for(Cf), self.gf_g, self.gf_b, self.part, silu=True, out_bf16=ws.af,
                      ldo=Cf)
        lib.gemm(ws.af, self.w_final, M=T, N=EMB, K=Cf, bias=self.b_final, out_f32=ws.y, w_static=True)
        for aw in self.attn:                                  # AttentionBlock without relative positions
            lib.groupnorm(ws.y, 1, T, EMB, _groups_for(EMB), aw.gn_g, aw.gn_b, self.part, out_bf16=ws.ay, ldo=EMB)
            lib.gemm(ws.ay, aw.wqkv, M=T, N=3 * EMB, K=EMB, bias=aw.bqkv, out_bf16=ws.qkv, w_static=True)
            # QKVAttentionLegacy scales q and k by ch^-1/4 each (arch_util.py:64-67)
            lib.attention(ws.qkv, ws.o, nseq=1, T=T, H=HEADS, ld=3 * EMB, ldo=EMB, k_off=EMB, v_off=2 * EMB,
                          scale=1.0 / math.sqrt(EMB // HEADS), head_dim=EMB // HEADS)
            lib.gemm(ws.o, aw.wproj, M=T, N=EMB, K=EMB, bias=aw.bproj, residual=ws.y, out_f32=ws.y, w_static=True)
        lib.linear_small(ws.y[0:1], 1, EMB, self.w_head, self.b_head, 2, ws.logits)

    def forward(self, clip):
        """clip: one waveform (any shape holding n samples) -> (logits fp32 [1, 2], softmax probabilities [1, 2]),
        both on the device."""
        wav = clip.reshape(-1).to(device=self.dev, dtype=torch.float32).contiguous()
        if wav.numel() < 1:
            raise ValueError("empty clip")
        ws = self.workspace(wav.numel())
        self.front(ws, wav)
        for l in range(DEPTH):
            self.level(ws, l)
        self.tail(ws)
        logits = ws.logits.clone()
        return logits, torch.softmax(logits, dim=-1)
