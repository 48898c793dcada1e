"""CVVP re-ranker on the sm_90a kernels (SURVEY §8f row 4: `tts(cvvp_amount > 0, voice_samples=...)`).

Mirrors `CVVP.forward(mel_cond, mel_codes, return_loss=False)` (tortoise/models/cvvp.py:108-124) as `tortoise/api.py:464-468`
accumulates it: the similarity of every candidate's mel codes to each conditioning clip, averaged over the clips. The
conditioning latent of a clip does not depend on the candidate (the reference repeats the clip for every row): it is
computed once per clip. Mean-pooling commutes with the last 1x1 convolution of `CollapsingTransformer.pre_combiner` and
with `to_*_latent`, so both run on the pooled `[n, D]` rows instead of on every position.
"""
import math

import torch

from . import lib
from .clvp_engine import _Encoder, encoder_layers
from .config import ModelConfig
from .diffusion_engine import _AttnW, _groups_for


def _bf(t, dev):
    return t.to(device=dev, dtype=torch.bfloat16).contiguous()


def _f(t, dev):
    return t.to(device=dev, dtype=torch.float32).contiguous()


class _Collapse:
    """CollapsingTransformer (cvvp.py:20-51) in eval mode."""

    def __init__(self, sd, p, D, H, depth, dev):
        self.enc = _Encoder(sd, p + "transformer.", depth, dev, wrap="")
        self.w0, self.b0 = _bf(sd[p + "pre_combiner.0.weight"].reshape(D, D), dev), _f(sd[p + "pre_combiner.0.bias"], dev)
        self.attn = _AttnW(sd, p + "pre_combiner.1.", D, H, dev)
        self.w2, self.b2 = _f(sd[p + "pre_combiner.2.weight"].reshape(D, D), dev), _f(sd[p + "pre_combiner.2.bias"], dev)


class CVVPEngine:
    def __init__(self, sd, cfg: ModelConfig, device="cuda"):
        self.cfg = cfg
        self.dev = torch.device(device)
        dev = self.dev
        D = self.D = cfg.cvvp_dim
        self.H = cfg.cvvp_heads
        self.groups = _groups_for(D)
        self.kpad = 128                                           # 80 mel channels padded to a multiple of 64
        w0 = torch.zeros(D // 2, 5, self.kpad)
        w0[:, :, :80] = sd["cond_emb.0.weight"].permute(0, 2, 1)  # [out, in, 5] -> [out, tap, in]
        self.w_c0, self.b_c0 = _bf(w0.reshape(D // 2, 5 * self.kpad), dev), _f(sd["cond_emb.0.bias"], dev)
        self.w_c1 = _bf(sd["cond_emb.1.weight"].permute(0, 2, 1).reshape(D, 3 * (D // 2)), dev)
        self.b_c1 = _f(sd["cond_emb.1.bias"], dev)
        self.speech_emb = _f(sd["speech_emb.emb.weight"], dev)
        self.w_cond_lat = _f(sd["to_conditioning_latent.weight"], dev)
        self.w_speech_lat = _f(sd["to_speech_latent.weight"], dev)
        self.temp_exp = float(math.exp(float(sd["temperature"])))
        self.cond = _Collapse(sd, "conditioning_transformer.", D, self.H, cfg.cvvp_depth, dev)
        self.speech = _Collapse(sd, "speech_transformer.", D, self.H, cfg.cvvp_depth, dev)

    # ------------------------------------------------------------------ CollapsingTransformer on x fp32 [nseq*T, D]
    def _collapse(self, cw, x, nseq, T):
        """-> pooled pre_combiner output fp32 [nseq, D] (before to_*_latent)."""
        D, H, dev = self.D, self.H, self.dev
        M = nseq * T
        encoder_layers(cw.enc, x, nseq, T, D, H, dev)
        a = torch.empty(M, D, dtype=torch.bfloat16, device=dev)
        lib.layernorm(x, M, D, cw.enc.norm_g, cw.enc.norm_b, out_bf16=a)         # ContinuousTransformerWrapper.norm
        y = torch.empty(M, D, dtype=torch.float32, device=dev)
        lib.gemm(a, cw.w0, M=M, N=D, K=D, bias=cw.b0, out_f32=y)                 # pre_combiner[0], Conv1d k=1
        # pre_combiner[1]: AttentionBlock without relative positions (arch_util.py:80-123), batched over the sequences
        aw = cw.attn
        lib.groupnorm(y, nseq, T, D, self.groups, aw.gn_g, aw.gn_b, lib.groupnorm_scratch(nseq, self.groups, dev),
                      out_bf16=a, ldo=D)
        qkv = torch.empty(M, 3 * D, dtype=torch.bfloat16, device=dev)
        lib.gemm(a, aw.wqkv, M=M, N=3 * D, K=D, bias=aw.bqkv, out_bf16=qkv)
        o = torch.empty(M, D, dtype=torch.bfloat16, device=dev)
        lib.attention(qkv, o, nseq=nseq, T=T, H=H, ld=3 * D, ldo=D, k_off=D, v_off=2 * D, scale=0.125)
        lib.gemm(o, aw.wproj, M=M, N=D, K=D, bias=aw.bproj, residual=y, out_f32=y)
        # mean over positions, then pre_combiner[2] (Conv1d k=1: affine, commutes with the mean)
        pooled = torch.empty(nseq, D, dtype=torch.float32, device=dev)
        for i in range(nseq):
            lib.mean_rows(y[i * T:(i + 1) * T], T, D, D, 1.0 / T, pooled[i])
        out = torch.empty(nseq, D, dtype=torch.float32, device=dev)
        lib.linear_small(pooled, nseq, D, cw.w2, cw.b2, D, out)
        return out

    def cond_latent(self, mel):
        """mel fp32 [80, Tm] (one clip of `auto_conds`) -> normalised conditioning latent [1, D] (cvvp.py:114-116)."""
        dev, D = self.dev, self.D
        mel = mel.to(dev).float().reshape(80, -1).contiguous()
        Tm = mel.shape[1]
        mt = torch.empty(Tm, 80, dtype=torch.float32, device=dev)
        lib.transpose_f32(mel, 80, Tm, mt)
        a0 = torch.empty(Tm, self.kpad, dtype=torch.bfloat16, device=dev)
        lib.cast_pad_bf16(mt, Tm, 80, 80, a0, self.kpad)
        # Conv1d(k, stride 2, padding k // 2) = every second row of the stride-1 convolution with the same padding
        y0 = torch.empty(Tm, D // 2, dtype=torch.float32, device=dev)
        lib.gemm(a0, self.w_c0, M=Tm, N=D // 2, K=self.kpad, taps=5, pad=2, bias=self.b_c0, out_f32=y0)
        T1 = (Tm + 1) // 2
        a1 = torch.empty(T1, D // 2, dtype=torch.bfloat16, device=dev)
        lib.cast_pad_bf16(y0, T1, D // 2, D, a1, D // 2)                         # rows 0, 2, 4, ...
        y1 = torch.empty(T1, D, dtype=torch.float32, device=dev)
        lib.gemm(a1, self.w_c1, M=T1, N=D, K=D // 2, taps=3, pad=1, bias=self.b_c1, out_f32=y1)
        T2 = (T1 + 1) // 2
        x = y1[0::2].contiguous()
        pooled = self._collapse(self.cond, x, 1, T2)
        lat = torch.empty(1, D, dtype=torch.float32, device=dev)
        lib.clvp_project(pooled, 1, D, self.w_cond_lat, lat, None, 1.0, None)
        return lat

    def scores(self, mels, codes, chunk=64):
        """≙ the accumulation of api.py:464-468 -> fp32 [B]. mels: tensor [1, n_clips, 80, Tm] (`auto_conds`) or a list
        of [80, Tm] / [1, 80, Tm]; codes int [B, L]."""
        dev, D = self.dev, self.D
        if torch.is_tensor(mels):
            mels = [mels[0, i] for i in range(mels.shape[1])]
        cond = torch.cat([self.cond_latent(m) for m in mels], dim=0)                    # [n_clips, D], unit rows
        # mean over clips of <s, c_i> = <s, mean_i c_i>
        cmean = torch.empty(D, dtype=torch.float32, device=dev)
        lib.mean_rows(cond, len(mels), D, D, 1.0 / len(mels), cmean)
        B, L = codes.shape
        codes = codes.to(device=dev, dtype=torch.int32).contiguous()
        if B * L > 0:
            lo, hi = int(codes.min().item()), int(codes.max().item())
            if lo < 0 or hi >= self.speech_emb.shape[0]:
                raise IndexError("CVVP speech token %d outside the embedding table [0, %d)" %
                                 (hi if hi >= self.speech_emb.shape[0] else lo, self.speech_emb.shape[0]))
        out = torch.empty(B, dtype=torch.float32, device=dev)
        for b0 in range(0, B, chunk):
            nb = min(chunk, B - b0)
            x = torch.empty(nb * L, D, dtype=torch.float32, device=dev)
            lib.embed(codes[b0:b0 + nb].reshape(-1), None, nb * L, D, self.speech_emb, None, x)
            pooled = self._collapse(self.speech, x, nb, L)
            lib.clvp_project(pooled, nb, D, self.w_speech_lat, None, cmean, self.temp_exp, out[b0:b0 + nb])
        return out
