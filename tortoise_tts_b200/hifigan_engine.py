"""HiFiGAN decoder of the reference's `api_fast` path on the sm_90a kernels (SURVEY §8f row 3).

Mirrors `HifiganGenerator.inference(gpt_latents, g=speaker_latent)` (tortoise/models/hifigan_decoder.py:270-294, forward
240-268, ResBlock1 83-97) as `api_fast.py:221-227` configures it: GPT latents [L, 1024] -> linear x 4 -> linear x 24000/22050
-> conv_pre(k 7) + cond_layer(speaker) -> 4 x [leaky_relu 0.1 -> ConvTranspose1d (x 8, 8, 2, 2) -> mean of three ResBlock1
(k 3 / 7 / 11, dilations 1 / 3 / 5)] -> leaky_relu (0.01) -> conv_post(k 7) -> tanh: 256 samples per input frame at 24 kHz.

Everything is token-major `[T, C]` and every convolution is one wgmma GEMM (`ttb_gemm`, conv taps = shifted TMA loads,
`tap_dilation` for the dilated ones):
  * operands are the error-compensated bf16 triple [hi | lo | hi] x [Wh | Wh | Wl] (fp32-grade products; a vocoder
    stacks ~45 convolutions and plain bf16 operands would not hold the 0.03 waveform tolerance), written by
    `ttb_act_split_cast`, which also applies the leaky_relu in front of every convolution and the mean over the three
    ResBlocks;
  * ConvTranspose1d(k = 2 s, stride s, padding s / 2) is a 3-tap GEMM with N = s x C_out: output sample q s + r sums two
    of the input rows q - 1, q, q + 1 (the third tap's weights are zero), and the `[T, s C_out]` result IS the token-major
    `[T s, C_out]` tensor;
  * the speaker conditioning `cond_layer(g)` is constant over time: folded into conv_pre's bias per call.
"""
import math

import torch

from . import lib
from .config import HIFI_LRELU, HIFI_RES_DILATIONS, HIFI_RES_KERNELS, HIFI_UP_FACTORS, ModelConfig


def _wn(sd, p):
    """weight_norm(dim=0) folded (hifigan_decoder.py:296-303 remove_weight_norm)."""
    v, g = sd[p + "weight_v"].float(), sd[p + "weight_g"].float()
    n = v.reshape(v.shape[0], -1).norm(dim=1).reshape(g.shape)
    return v * (g / n)


def _kt(C):
    """K per tap of the split operand [hi | lo | hi]: 3 C columns rounded up to the GEMM's K block (64)."""
    return ((3 * C + 63) // 64) * 64


def _pack_conv(w, dev):
    """Conv1d weight [out, in, k] -> bf16 [out, k * Kt] with [Wh | Wh | Wl | 0] per tap."""
    out_c, in_c, k = w.shape
    kt = _kt(in_c)
    wt = w.permute(0, 2, 1).contiguous()                  # [out, tap, in]
    hi = wt.to(torch.bfloat16)
    lo = (wt - hi.float()).to(torch.bfloat16)
    pk = torch.zeros(out_c, k, kt, dtype=torch.bfloat16)
    pk[:, :, :in_c], pk[:, :, in_c:2 * in_c], pk[:, :, 2 * in_c:3 * in_c] = hi, hi, lo
    return pk.reshape(out_c, k * kt).to(dev).contiguous()


def _convt_as_conv(w, s):
    """ConvTranspose1d weight [in, out, 2 s] (stride s, padding s / 2) -> the equivalent 3-tap Conv1d weight
    [s * out, in, 3] on rows (q - 1, q, q + 1): output sample q s + r, channel co = column r * out + co."""
    in_c, out_c, k = w.shape
    assert k == 2 * s and s % 2 == 0
    p = s // 2
    g = torch.zeros(s * out_c, in_c, 3)
    for r in range(s):
        rows = slice(r * out_c, (r + 1) * out_c)
        if r + p < s:          # input rows q (k = r + p) and q - 1 (k = r + p + s)
            g[rows, :, 1] = w[:, :, r + p].t()
            g[rows, :, 0] = w[:, :, r + p + s].t()
        else:                  # input rows q + 1 (k = r + p - s) and q (k = r + p)
            g[rows, :, 2] = w[:, :, r + p - s].t()
            g[rows, :, 1] = w[:, :, r + p].t()
    return g


class HifiganEngine:
    def __init__(self, sd, cfg: ModelConfig, device="cuda"):
        self.cfg = cfg
        self.dev = torch.device(device)
        dev = self.dev
        self.D, self.C0 = cfg.ar_dim, cfg.hifi_channels
        f = lambda t: t.to(device=dev, dtype=torch.float32).contiguous()      # noqa: E731
        self.w_pre = _pack_conv(_wn(sd, "conv_pre."), dev)
        # cond_layer(g) + conv_pre.bias = one bias vector per call
        self.w_cond = f(sd["cond_layer.weight"].reshape(self.C0, self.D))
        self.b_cond = f(sd["cond_layer.bias"] + sd["conv_pre.bias"])
        self.ups, self.res = [], []
        ch = self.C0
        for i, u in enumerate(HIFI_UP_FACTORS):
            w = _convt_as_conv(_wn(sd, f"ups.{i}."), u)
            self.ups.append((_pack_conv(w, dev), f(sd[f"ups.{i}.bias"].repeat(u)), ch, u))
            ch //= 2
            blocks = []
            for j, k in enumerate(HIFI_RES_KERNELS):
                p = f"resblocks.{i * len(HIFI_RES_KERNELS) + j}."
                convs = []
                for m, d in enumerate(HIFI_RES_DILATIONS):
                    convs.append((_pack_conv(_wn(sd, p + f"convs1.{m}."), dev), f(sd[p + f"convs1.{m}.bias"]),
                                  _pack_conv(_wn(sd, p + f"convs2.{m}."), dev), f(sd[p + f"convs2.{m}.bias"]), d))
                blocks.append((k, convs))
            self.res.append(blocks)
        self.w_post = _pack_conv(_wn(sd, "conv_post."), dev)
        self.b_post = f(sd["conv_post.bias"])
        self.c_last = ch

    @staticmethod
    def output_frames(L):
        """Frames after the two interpolations of `inference` (hifigan_decoder.py:283-292); 256 samples each."""
        return int(math.floor(int(math.floor(L * 4.0)) * (24000 / 22050)))

    def _split(self, a, R, C, slope=1.0, b=None, c=None, scale=1.0):
        out = torch.empty(R, _kt(C), dtype=torch.bfloat16, device=self.dev)
        lib.act_split_cast(a, R, C, out, _kt(C), b=b, c=c, scale=scale, slope=slope)
        return out

    def _conv(self, a, w, bias, T, cin, cout, k, dil=1, residual=None, out=None, act=lib.ACT_NONE):
        out = torch.empty(T, cout, dtype=torch.float32, device=self.dev) if out is None else out
        tile = 32 if cout <= 32 else (64 if cout <= 64 else 0)
        lib.gemm(a, w, M=T, N=cout, K=_kt(cin), taps=k, pad=dil * (k - 1) // 2, tap_dilation=dil, bias=bias,
                 residual=residual, out_f32=out, act=act, tile_n=tile)
        return out

    def inference(self, latents, speaker):
        """latents fp32 [L, D] (GPT latents of ONE utterance), speaker fp32 [D] (auto conditioning latent)
        -> waveform fp32 [256 * output_frames(L)] in [-1, 1]."""
        dev, D = self.dev, self.D
        lat = latents.to(dev).float().reshape(-1, D).contiguous()
        L = lat.shape[0]
        T1 = int(math.floor(L * 4.0))
        T = self.output_frames(L)
        up1 = torch.empty(T1, D, dtype=torch.float32, device=dev)
        lib.interp_linear(lat, L, D, 1.0 / 4.0, T1, up1)
        up2 = torch.empty(T, D, dtype=torch.float32, device=dev)
        lib.interp_linear(up1, T1, D, 22050.0 / 24000.0, T, up2)
        bias_pre = torch.empty(self.C0, dtype=torch.float32, device=dev)
        lib.linear_small(speaker.to(dev).float().reshape(1, D).contiguous(), 1, D, self.w_cond, self.b_cond, self.C0, bias_pre)
        o = self._conv(self._split(up2, T, D), self.w_pre, bias_pre, T, D, self.C0, 7)
        a = self._split(o, T, self.C0, slope=HIFI_LRELU)                      # leaky_relu before ups[0]
        for i, (w_up, b_up, ch, u) in enumerate(self.ups):
            co = ch // 2
            o = self._conv(a, w_up, b_up, T, ch, u * co, 3)                    # [T, u * co] == [T * u, co]
            T *= u
            streams = []
            for k, convs in self.res[i]:
                x = o                                                          # ResBlock1 input (shared by the three)
                for m, (w1, b1, w2, b2, d) in enumerate(convs):
                    t = self._conv(self._split(x, T, co, slope=HIFI_LRELU), w1, b1, T, co, co, k, dil=d)
                    xn = torch.empty(T, co, dtype=torch.float32, device=dev) if m == 0 else x
                    self._conv(self._split(t, T, co, slope=HIFI_LRELU), w2, b2, T, co, co, k, residual=x, out=xn)
                    x = xn
                streams.append(x)
            # o = mean of the three ResBlocks, then the leaky_relu in front of the next layer (0.1, or F.leaky_relu's
            # default 0.01 before conv_post, hifigan_decoder.py:265)
            last = i == len(self.ups) - 1
            a = self._split(streams[0], T, co, slope=0.01 if last else HIFI_LRELU, b=streams[1], c=streams[2],
                            scale=1.0 / len(streams))
        wav = torch.empty(T, 1, dtype=torch.float32, device=dev)
        self._conv(a, self.w_post, self.b_post, T, self.c_last, 1, 7, out=wav, act=lib.ACT_TANH)
        return wav.reshape(-1)
