"""wav2vec2 CTC aligner on the sm_90a kernels: the Wav2Vec2ForCTC forward that `Wav2VecAlignment.align` runs
(utils/wav2vec_alignment.py:53,61-70) to find where each character of the text is spoken.

    wav 24 kHz -> resample to 16 kHz (torchaudio, :64) -> (x - mean) / sqrt(var + 1e-7) (:65)
      -> feature extractor: 7 x {Conv1d, LayerNorm over channels, GELU}      (HF Wav2Vec2LayerNormConvLayer)
      -> feature projection: LayerNorm, Linear(C -> H)
      -> + GELU(grouped positional Conv1d) (weight norm folded at load, last frame dropped: SamePad)
      -> L x pre-LN encoder layer {x += attn(LN(x)); x += FF(LN(x))} -> LayerNorm -> lm_head -> logits [T, V]

Strided convs 1-6 run as ttb_gemm over a PAIR VIEW of their input: rows [L, C] read as [ceil(L/2), 2C], so a stride-2
conv is a stride-1 GEMM: k = 2 is one tap [W0|W1]; k = 3 is two taps [W0|W1] and [W2|0]. One zero row after the input
keeps the second half of the last pair defined when L is odd. Only checkpoints of this architecture are accepted
(`check_config`); anything else is rejected with the reason.
"""
import json
import math
import os

import torch

from . import lib
from .conditioning_engine import _resample_kernels

CONV_KERNELS = (10, 3, 3, 3, 3, 2, 2)
CONV_STRIDES = (5, 2, 2, 2, 2, 2, 2)
SAMPLE_RATE = 24000            # the rate of the waveforms tts() returns (Wav2VecAlignment.align's audio_sample_rate)
MODEL_RATE = 16000


def check_config(cfg):
    """Raise ValueError unless `cfg` (an HF Wav2Vec2Config as a dict) describes the architecture this engine runs.
    Missing keys take the Wav2Vec2Config defaults."""
    g = cfg.get
    bad = []
    if not g("do_stable_layer_norm", False):
        bad.append("do_stable_layer_norm must be true (pre-LayerNorm encoder)")
    if g("feat_extract_norm", "group") != "layer":
        bad.append("feat_extract_norm must be 'layer'")
    if not g("conv_bias", False):
        bad.append("conv_bias must be true")
    for k in ("feat_extract_activation", "hidden_act"):
        if g(k, "gelu") != "gelu":
            bad.append("%s must be 'gelu'" % k)
    if tuple(g("conv_kernel", ())) != CONV_KERNELS or tuple(g("conv_stride", ())) != CONV_STRIDES:
        bad.append("conv_kernel / conv_stride must be %s / %s" % (list(CONV_KERNELS), list(CONV_STRIDES)))
    dims = list(g("conv_dim", [512] * 7))
    if len(set(dims)) != 1 or dims[0] % 128 or dims[0] > 512:
        bad.append("conv_dim must be 7 equal widths, a multiple of 128 and <= 512 (got %s)" % dims)
    H, nh = g("hidden_size", 768), g("num_attention_heads", 12)
    if H != 64 * nh or H % 128:
        bad.append("hidden_size must be 64 * num_attention_heads and a multiple of 128")
    groups = g("num_conv_pos_embedding_groups", 16)
    if H % groups or (H // groups) % 64:
        bad.append("hidden_size / num_conv_pos_embedding_groups must be a multiple of 64")
    if g("intermediate_size", 3072) % 64:
        bad.append("intermediate_size must be a multiple of 64")
    if abs(g("layer_norm_eps", 1e-5) - 1e-5) > 1e-12:
        bad.append("layer_norm_eps must be 1e-5")
    if g("add_adapter", False) or g("adapter_attn_dim", None) is not None:
        bad.append("adapters are not supported")
    if bad:
        raise ValueError("unsupported wav2vec2 checkpoint: " + "; ".join(bad))


def load_checkpoint(model_dir):
    """HF-format checkpoint directory -> (config dict, state dict): config.json plus model.safetensors or
    pytorch_model.bin."""
    with open(os.path.join(model_dir, "config.json")) as f:
        cfg = json.load(f)
    st = os.path.join(model_dir, "model.safetensors")
    if os.path.exists(st):
        from safetensors.torch import load_file
        sd = load_file(st)
    else:
        pt = os.path.join(model_dir, "pytorch_model.bin")
        if not os.path.exists(pt):
            raise FileNotFoundError("%s has neither model.safetensors nor pytorch_model.bin" % model_dir)
        sd = torch.load(pt, map_location="cpu", weights_only=True)
    return cfg, sd


def _pos_conv_weight(sd, prefix):
    """The positional conv's weight with its weight norm (dim = 2) folded; both state-dict forms."""
    if prefix + "weight_g" in sd:
        g, v = sd[prefix + "weight_g"], sd[prefix + "weight_v"]
    elif prefix + "parametrizations.weight.original0" in sd:
        g, v = sd[prefix + "parametrizations.weight.original0"], sd[prefix + "parametrizations.weight.original1"]
    else:
        return sd[prefix + "weight"].float()
    return torch._weight_norm(v.float(), g.float(), 2)


class _Workspace:
    """Every buffer of one forward at one input length (allocated once per length)."""

    def __init__(self, eng, n24):
        dev, C, H = eng.dev, eng.C, eng.H
        self.n24 = n24
        self.n16 = -(-MODEL_RATE * n24 // SAMPLE_RATE)               # torchaudio: ceil(new * n / orig)
        lens = [(self.n16 - CONV_KERNELS[0]) // CONV_STRIDES[0] + 1]
        for k, s in zip(CONV_KERNELS[1:], CONV_STRIDES[1:]):
            lens.append((lens[-1] - k) // s + 1)
        if lens[-1] < 1:
            raise ValueError("clip too short for the aligner: %d samples at 24 kHz" % n24)
        self.lens = lens
        self.T = T = lens[-1]
        f32, bf = dict(dtype=torch.float32, device=dev), dict(dtype=torch.bfloat16, device=dev)
        self.x16 = torch.empty(self.n16, **f32)
        self.stats = torch.empty(2, **f32)
        # feature maps ping-pong between two bf16 buffers; row L after an L-row map is kept zero (pair view)
        self.fbuf = [torch.zeros(lens[0] + 1, C, **bf), torch.zeros(lens[1] + 1, C, **bf)]
        self.y = torch.empty(lens[1], C, **f32)
        self.feat = torch.empty(T, C, **f32)
        self.pn = torch.empty(T, C, **bf)
        self.x = torch.empty(T, H, **f32)
        self.xb = torch.empty(T, H, **bf)
        self.a = torch.empty(T, H, **bf)
        self.qkv = torch.empty(T, 3 * H, **bf)
        self.o = torch.empty(T, H, **bf)
        self.h = torch.empty(T, eng.FF, **bf)
        self.logits = torch.empty(T, eng.V, **f32)
        self.ids = torch.empty(T, dtype=torch.int32, device=dev)


class Wav2VecEngine:
    def __init__(self, config, state_dict, device="cuda"):
        check_config(config)
        self.dev = dev = torch.device(device)
        sd = state_dict
        p = "wav2vec2."
        self.C = C = config.get("conv_dim", [512] * 7)[0]
        self.H = H = config["hidden_size"]
        self.heads = config["num_attention_heads"]
        self.FF = config["intermediate_size"]
        self.L = config["num_hidden_layers"]
        self.V = sd["lm_head.weight"].shape[0]
        self.groups = config.get("num_conv_pos_embedding_groups", 16)
        self.pos_k = config.get("num_conv_pos_embeddings", 128)

        def f(t):
            return t.to(device=dev, dtype=torch.float32).contiguous()

        def bf(t):
            return t.to(device=dev, dtype=torch.bfloat16).contiguous()
        k, self.rs_down, self.rs_up, self.rs_width = _resample_kernels(SAMPLE_RATE, MODEL_RATE)
        self.rs_kernels = k.to(dev)
        fe = p + "feature_extractor.conv_layers."
        self.conv = []
        for i, kk in enumerate(CONV_KERNELS):
            w = sd[fe + f"{i}.conv.weight"].float()                   # [C_out, C_in, k]
            if i == 0:
                wp = f(w.reshape(C, kk))
            else:                                                    # pair view: [W0|W1] (+ [W2|0]) per output row
                taps = (kk + 1) // 2
                wk = torch.zeros(C, 2 * taps, C)
                wk[:, :kk] = w.permute(0, 2, 1)
                wp = bf(wk.reshape(C, taps * 2 * C))
            self.conv.append((wp, f(sd[fe + f"{i}.conv.bias"]), f(sd[fe + f"{i}.layer_norm.weight"]),
                              f(sd[fe + f"{i}.layer_norm.bias"])))
        fp = p + "feature_projection."
        self.fp_g, self.fp_b = f(sd[fp + "layer_norm.weight"]), f(sd[fp + "layer_norm.bias"])
        self.w_proj, self.b_proj = bf(sd[fp + "projection.weight"]), f(sd[fp + "projection.bias"])
        pc = p + "encoder.pos_conv_embed.conv."
        wpos = _pos_conv_weight(sd, pc)                               # [H, H / groups, k]
        Hg = H // self.groups
        self.w_pos = [bf(wpos[g * Hg:(g + 1) * Hg].permute(0, 2, 1).reshape(Hg, self.pos_k * Hg))
                      for g in range(self.groups)]
        self.b_pos = f(sd[pc + "bias"])
        self.layers = []
        for l in range(self.L):
            q = p + f"encoder.layers.{l}."
            a = q + "attention."
            self.layers.append(dict(
                ln1_g=f(sd[q + "layer_norm.weight"]), ln1_b=f(sd[q + "layer_norm.bias"]),
                wqkv=bf(torch.cat([sd[a + n + "_proj.weight"] for n in "qkv"], 0)),
                bqkv=f(torch.cat([sd[a + n + "_proj.bias"] for n in "qkv"], 0)),
                wo=bf(sd[a + "out_proj.weight"]), bo=f(sd[a + "out_proj.bias"]),
                ln2_g=f(sd[q + "final_layer_norm.weight"]), ln2_b=f(sd[q + "final_layer_norm.bias"]),
                w1=bf(sd[q + "feed_forward.intermediate_dense.weight"]), b1=f(sd[q + "feed_forward.intermediate_dense.bias"]),
                w2=bf(sd[q + "feed_forward.output_dense.weight"]), b2=f(sd[q + "feed_forward.output_dense.bias"])))
        self.enc_g, self.enc_b = f(sd[p + "encoder.layer_norm.weight"]), f(sd[p + "encoder.layer_norm.bias"])
        self.w_head, self.b_head = bf(sd["lm_head.weight"]), f(sd["lm_head.bias"])
        self._ws = {}

    def _workspace(self, n24):
        ws = self._ws.get(n24)
        if ws is None:
            if len(self._ws) >= 4:           # candidates of one call share a few lengths; do not grow without bound
                self._ws.clear()
            ws = self._ws[n24] = _Workspace(self, n24)
        return ws

    def _forward(self, wav24k):
        wav = wav24k.reshape(-1).to(device=self.dev, dtype=torch.float32).contiguous()
        ws = self._workspace(wav.numel())
        C, H, T = self.C, self.H, ws.T
        lib.audio_resample(wav, ws.n24, self.rs_kernels, self.rs_down, self.rs_up, self.rs_kernels.shape[1],
                           self.rs_width, ws.x16, ws.n16)
        w0, b0, g0, be0 = self.conv[0]
        lib.wav2vec_conv0(ws.x16, ws.n16, w0, b0, g0, be0, C, ws.stats, ws.fbuf[0], C)
        for i in range(1, len(CONV_KERNELS)):
            src, dst = ws.fbuf[(i - 1) % 2], ws.fbuf[i % 2]
            Lin, Lout = ws.lens[i - 1], ws.lens[i]
            w, b, g, be = self.conv[i]
            taps = (CONV_KERNELS[i] + 1) // 2
            lib.gemm(src, w, M=Lout, N=C, K=2 * C, rows=(Lin + 1) // 2, taps=taps, bias=b, out_f32=ws.y, w_static=True)
            last = i == len(CONV_KERNELS) - 1
            lib.layernorm_act(ws.y, Lout, C, g, be, gelu=True, out_bf16=None if last else dst,
                              out_f32=ws.feat if last else None)
            if not last:
                dst[Lout].zero_()
        lib.layernorm(ws.feat, T, C, self.fp_g, self.fp_b, out_bf16=ws.pn)
        lib.gemm(ws.pn, self.w_proj, M=T, N=H, K=C, bias=self.b_proj, out_f32=ws.x, out_bf16=ws.xb, w_static=True)
        Hg = H // self.groups
        for g in range(self.groups):                   # grouped conv: one GEMM per group, x += GELU(conv(x))
            cs = slice(g * Hg, (g + 1) * Hg)
            lib.gemm(ws.xb[:, cs], self.w_pos[g], M=T, N=Hg, K=Hg, lda=H, taps=self.pos_k, pad=self.pos_k // 2,
                     bias=self.b_pos[cs], act=lib.ACT_GELU_ERF, residual=ws.x[:, cs], ldr=H, out_f32=ws.x[:, cs], ldo=H,
                     w_static=True)
        for lw in self.layers:
            lib.layernorm(ws.x, T, H, lw["ln1_g"], lw["ln1_b"], out_bf16=ws.a)
            lib.gemm(ws.a, lw["wqkv"], M=T, N=3 * H, K=H, bias=lw["bqkv"], out_bf16=ws.qkv, w_static=True)
            lib.attention(ws.qkv, ws.o, nseq=1, T=T, H=self.heads, ld=3 * H, ldo=H, k_off=H, v_off=2 * H,
                          scale=1.0 / math.sqrt(64))
            lib.gemm(ws.o, lw["wo"], M=T, N=H, K=H, bias=lw["bo"], residual=ws.x, out_f32=ws.x, w_static=True)
            lib.layernorm(ws.x, T, H, lw["ln2_g"], lw["ln2_b"], out_bf16=ws.a)
            lib.gemm(ws.a, lw["w1"], M=T, N=self.FF, K=H, bias=lw["b1"], act=lib.ACT_GELU_ERF, out_bf16=ws.h,
                     w_static=True)
            lib.gemm(ws.h, lw["w2"], M=T, N=H, K=self.FF, bias=lw["b2"], residual=ws.x, out_f32=ws.x, w_static=True)
        lib.layernorm(ws.x, T, H, self.enc_g, self.enc_b, out_bf16=ws.a)
        lib.gemm(ws.a, self.w_head, M=T, N=self.V, K=H, bias=self.b_head, out_f32=ws.logits, w_static=True)
        return ws

    def logits(self, wav24k):
        """wav24k: waveform at 24 kHz (any shape holding one clip) -> fp32 logits [T, V] on the device."""
        return self._forward(wav24k).logits.clone()

    def ids(self, wav24k):
        """-> int32 [T] on the device: the argmax token of every frame."""
        ws = self._forward(wav24k)
        lib.argmax_rows(ws.logits, ws.T, self.V, ws.ids)
        return ws.ids.clone()
