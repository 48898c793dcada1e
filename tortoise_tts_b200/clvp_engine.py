"""CLVP re-ranker on the sm_90a kernels (SURVEY §8 row a5).

Mirrors `CLVP.forward(text, speech_tokens, return_loss=False)` (tortoise/models/clvp.py:99-140) for the
x-transformers Encoder configuration the reference builds (clvp.py:54-83). The text latent is computed ONCE per
utterance instead of once per candidate (the reference repeats the text for every row, api.py:463).
"""
import math

import torch

from . import lib
from .config import ModelConfig


def _bf(t, dev):
    return t.to(device=dev, dtype=torch.bfloat16).contiguous()


def _f(t, dev):
    return t.to(device=dev, dtype=torch.float32).contiguous()


class _Encoder:
    """Weights of one x-transformers Encoder. `wrap`: "wrap." for CLVP's CheckpointedXTransformerEncoder keys
    (arch_util.py:334-373), "" for a plain ContinuousTransformerWrapper (CVVP, cvvp.py:23-36)."""

    def __init__(self, sd, prefix, depth, dev, wrap="wrap."):
        self.layers = []
        for l in range(depth):
            a = f"{prefix}attn_layers.layers.{2 * l}."
            f = f"{prefix}attn_layers.layers.{2 * l + 1}."
            wq, wk, wv = (sd[a + f"1.{wrap}{n}.weight"] for n in ("to_q", "to_k", "to_v"))
            w1, b1 = sd[f + f"1.{wrap}net.0.proj.weight"], sd[f + f"1.{wrap}net.0.proj.bias"]
            inner = w1.shape[0] // 2
            self.inner = inner
            # GLU: x, gate = proj(x).chunk(2) (xtransformers.py:435-437) -> interleave rows (u0,g0,u1,g1,...) so the
            # GEMM epilogue can form u*gelu(g) from adjacent accumulator columns
            w1i = torch.stack([w1[:inner], w1[inner:]], dim=1).reshape(2 * inner, -1)
            b1i = torch.stack([b1[:inner], b1[inner:]], dim=1).reshape(2 * inner)
            self.layers.append(dict(
                g_attn=_f(sd[a + "0.0.g"], dev), wqkv=_bf(torch.cat([wq, wk, wv], dim=0), dev),
                wout=_bf(sd[a + f"1.{wrap}to_out.weight"], dev), bout=_f(sd[a + f"1.{wrap}to_out.bias"], dev),
                g_ff=_f(sd[f + "0.0.g"], dev), w1=_bf(w1i, dev), b1=_f(b1i, dev),
                w2=_bf(sd[f + f"1.{wrap}net.3.weight"], dev), b2=_f(sd[f + f"1.{wrap}net.3.bias"], dev)))
        self.norm_g = _f(sd[prefix + "norm.weight"], dev)
        self.norm_b = _f(sd[prefix + "norm.bias"], dev)


def encoder_layers(enc, x, nseq, T, D, H, dev):
    """The Encoder's layer stack on the fp32 residual stream x [nseq*T, D], in place (everything but the final
    LayerNorm): pre-RMSNorm attention with rotary 32 on q / k / v, pre-RMSNorm GEGLU feed-forward
    (xtransformers.py:906-1013 as configured in clvp.py:54-83 and cvvp.py:23-36)."""
    M = nseq * T
    a = torch.empty(M, D, dtype=torch.bfloat16, device=dev)
    qkv = torch.empty(M, 3 * D, dtype=torch.bfloat16, device=dev)
    o = torch.empty(M, D, dtype=torch.bfloat16, device=dev)
    h = torch.empty(M, enc.inner, dtype=torch.bfloat16, device=dev)
    for lw in enc.layers:
        lib.rmsnorm(x, M, D, lw["g_attn"], a)
        lib.gemm(a, lw["wqkv"], M=M, N=3 * D, K=D, out_bf16=qkv)
        lib.clvp_rotary(qkv, nseq, T, H)
        lib.attention(qkv, o, nseq=nseq, T=T, H=H, ld=3 * D, ldo=D, k_off=D, v_off=2 * D, scale=0.125)
        lib.gemm(o, lw["wout"], M=M, N=D, K=D, bias=lw["bout"], residual=x, out_f32=x)
        lib.rmsnorm(x, M, D, lw["g_ff"], a)
        lib.gemm(a, lw["w1"], M=M, N=2 * enc.inner, K=D, bias=lw["b1"], act=lib.ACT_GEGLU, out_bf16=h)
        lib.gemm(h, lw["w2"], M=M, N=D, K=enc.inner, bias=lw["b2"], residual=x, out_f32=x)


class CLVPEngine:
    def __init__(self, sd, cfg: ModelConfig, device="cuda"):
        self.cfg = cfg
        self.dev = torch.device(device)
        dev = self.dev
        self.D, self.H = cfg.clvp_dim, cfg.clvp_heads
        self.text_emb = _f(sd["text_emb.weight"], dev)
        self.speech_emb = _f(sd["speech_emb.weight"], dev)
        self.w_text_lat = _f(sd["to_text_latent.weight"], dev)
        self.w_speech_lat = _f(sd["to_speech_latent.weight"], dev)
        self.temp_exp = float(math.exp(float(sd["temperature"])))
        self.text_enc = _Encoder(sd, "text_transformer.transformer.", cfg.clvp_depth, dev)
        self.speech_enc = _Encoder(sd, "speech_transformer.transformer.", cfg.clvp_depth, dev)

    def _encode(self, enc, ids, table, nseq, T):
        """ids int32 [nseq*T] -> pooled LayerNorm'd mean [nseq, D]."""
        D, dev = self.D, self.dev
        M = nseq * T
        x = torch.empty(M, D, dtype=torch.float32, device=dev)
        lib.embed(ids, None, M, D, table, None, x)
        encoder_layers(enc, x, nseq, T, D, self.H, dev)
        pooled = torch.empty(nseq, D, dtype=torch.float32, device=dev)
        lib.clvp_pool(x, nseq, T, D, enc.norm_g, enc.norm_b, pooled)
        return pooled

    def text_latent(self, text_tokens):
        dev = self.dev
        ids = torch.as_tensor([int(v) for v in text_tokens], dtype=torch.int32, device=dev)
        pooled = self._encode(self.text_enc, ids, self.text_emb, 1, ids.numel())
        lat = torch.empty(1, self.D, dtype=torch.float32, device=dev)
        lib.clvp_project(pooled, 1, self.D, self.w_text_lat, lat, None, 1.0, None)
        return lat

    def scores(self, text_tokens, codes, chunk=64):
        """≙ clvp(text.repeat(B,1), codes, return_loss=False) -> fp32 [B]. codes int [B, L]."""
        dev = self.dev
        B, L = codes.shape
        tl = self.text_latent(text_tokens)
        out = torch.empty(B, dtype=torch.float32, device=dev)
        codes = codes.to(device=dev, dtype=torch.int32).contiguous()
        # the embedding gather is unchecked on the device: an id outside the table (the AR vocabulary has two ids more
        # than speech_emb: start 8192 / stop 8193) raises here as nn.Embedding does in the reference (clvp.py:114)
        if B * L > 0:
            lo, hi = int(codes.min().item()), int(codes.max().item())
            if lo < 0 or hi >= self.speech_emb.shape[0]:
                raise IndexError("CLVP speech token %d outside the embedding table [0, %d)" %
                                 (hi if hi >= self.speech_emb.shape[0] else lo, self.speech_emb.shape[0]))
        if any(int(t) < 0 or int(t) >= self.text_emb.shape[0] for t in text_tokens):
            raise IndexError("CLVP text token outside the embedding table [0, %d)" % self.text_emb.shape[0])
        for b0 in range(0, B, chunk):
            nb = min(chunk, B - b0)
            pooled = self._encode(self.speech_enc, codes[b0:b0 + nb].reshape(-1), self.speech_emb, nb, L)
            lib.clvp_project(pooled, nb, self.D, self.w_speech_lat, None, tl, self.temp_exp, out[b0:b0 + nb])
        return out
