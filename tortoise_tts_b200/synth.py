"""Synthetic checkpoints in the reference's `.pth` layout (SURVEY.md App. B / §8d "Weights").

No trained weights are reachable offline, so benchmarks and parity tests run on seeded
random weights with exactly the tensor names/shapes the reference modules produce
(`tortoise/api.py:217-238`).  Nothing here instantiates a reference module: the names are
generated from the layout; `oracle/ref_build.py` (used by `tests/test_oracle_vs_reference.py` in the build container,
where the reference is importable) loads them into the reference modules with `strict=True`, and
`tests/test_host_logic.py::test_synth_layout_param_counts` checks the parameter counts of SURVEY App. B anywhere.

Conventions (SURVEY.md §8d): zero-initialised tensors of the reference (AttentionBlock.proj_out,
arch_util.py:111) are drawn N(0, .02) so attention is exercised; norm affines are jittered;
with `suppress_stop=True` `mel_head.bias[8192:8194] = -1e4` so no candidate emits the start or
stop token and every candidate runs exactly `max_mel_tokens` steps (deterministic audio length).
"""
import math
import os

import torch

from .config import ModelConfig, VOC_STRIDES, VOC_DILATIONS


class _Gen:
    def __init__(self, seed):
        self.g = torch.Generator(device="cpu")
        self.g.manual_seed(seed)

    def normal(self, shape, std):
        return torch.randn(shape, generator=self.g, dtype=torch.float32) * std

    def lin(self, shape, fan_in, gain=1.0):
        return self.normal(shape, gain / math.sqrt(fan_in))

    def gamma(self, n):
        return 1.0 + self.normal((n,), 0.1)

    def beta(self, n):
        return self.normal((n,), 0.1)

    def bias(self, n, std=0.02):
        return self.normal((n,), std)


def _attention_block(sd, g, prefix, C, heads, rel_pos):
    """AttentionBlock (arch_util.py:80-123)."""
    sd[prefix + "norm.weight"] = g.gamma(C)
    sd[prefix + "norm.bias"] = g.beta(C)
    sd[prefix + "qkv.weight"] = g.lin((3 * C, C, 1), C)
    sd[prefix + "qkv.bias"] = g.bias(3 * C)
    sd[prefix + "proj_out.weight"] = g.lin((C, C, 1), C, 0.5)
    sd[prefix + "proj_out.bias"] = g.bias(C)
    if rel_pos:
        sd[prefix + "relative_pos_embeddings.relative_attention_bias.weight"] = g.normal((32, heads), 0.5)


def synth_autoregressive(cfg: ModelConfig, seed=0, suppress_stop=True):
    """`autoregressive.pth` (UnifiedVoice.state_dict(), autoregressive.py:293-357)."""
    g = _Gen(seed * 1000 + 1)
    D = cfg.ar_dim
    sd = {}
    sd["conditioning_encoder.init.weight"] = g.lin((D, 80, 1), 80)
    sd["conditioning_encoder.init.bias"] = g.bias(D)
    for i in range(cfg.cond_enc_blocks):
        _attention_block(sd, g, f"conditioning_encoder.attn.{i}.", D, cfg.ar_heads, False)
    sd["text_embedding.weight"] = g.normal((cfg.number_text_tokens + 1, D), 0.02)
    sd["mel_embedding.weight"] = g.normal((cfg.number_mel_codes, D), 0.02)
    for l in range(cfg.ar_layers):
        p = f"gpt.h.{l}."
        sd[p + "ln_1.weight"] = g.gamma(D)
        sd[p + "ln_1.bias"] = g.beta(D)
        sd[p + "attn.c_attn.weight"] = g.lin((D, 3 * D), D)          # HF Conv1D: [in, out]
        sd[p + "attn.c_attn.bias"] = g.bias(3 * D)
        sd[p + "attn.c_proj.weight"] = g.lin((D, D), D, 0.5)
        sd[p + "attn.c_proj.bias"] = g.bias(D)
        sd[p + "ln_2.weight"] = g.gamma(D)
        sd[p + "ln_2.bias"] = g.beta(D)
        sd[p + "mlp.c_fc.weight"] = g.lin((D, 4 * D), D)
        sd[p + "mlp.c_fc.bias"] = g.bias(4 * D)
        sd[p + "mlp.c_proj.weight"] = g.lin((4 * D, D), 4 * D, 0.5)
        sd[p + "mlp.c_proj.bias"] = g.bias(D)
    sd["gpt.ln_f.weight"] = g.gamma(D)
    sd["gpt.ln_f.bias"] = g.beta(D)
    sd["mel_pos_embedding.emb.weight"] = g.normal((cfg.mel_pos_rows, D), 0.02)
    sd["text_pos_embedding.emb.weight"] = g.normal((cfg.text_pos_rows, D), 0.02)
    sd["final_norm.weight"] = g.gamma(D)
    sd["final_norm.bias"] = g.beta(D)
    sd["text_head.weight"] = g.lin((cfg.number_text_tokens + 1, D), D)
    sd["text_head.bias"] = g.bias(cfg.number_text_tokens + 1)
    # logits of scale ~3 so that top-p sampling has a non-trivial nucleus
    sd["mel_head.weight"] = g.lin((cfg.number_mel_codes, D), D, 3.0)
    sd["mel_head.bias"] = g.bias(cfg.number_mel_codes)
    if suppress_stop:
        sd["mel_head.bias"][cfg.start_mel_token] = -1e4
        sd["mel_head.bias"][cfg.stop_mel_token] = -1e4
    return sd


def _diff_resblock(sd, g, prefix, C):
    """ResBlock (diffusion_decoder.py:60-120), efficient_config: in conv k=1, out conv k=3."""
    sd[prefix + "in_layers.0.weight"] = g.gamma(C)
    sd[prefix + "in_layers.0.bias"] = g.beta(C)
    sd[prefix + "in_layers.2.weight"] = g.lin((C, C, 1), C)
    sd[prefix + "in_layers.2.bias"] = g.bias(C)
    sd[prefix + "emb_layers.1.weight"] = g.lin((2 * C, C), C, 0.3)
    sd[prefix + "emb_layers.1.bias"] = g.bias(2 * C)
    sd[prefix + "out_layers.0.weight"] = g.gamma(C)
    sd[prefix + "out_layers.0.bias"] = g.beta(C)
    sd[prefix + "out_layers.3.weight"] = g.lin((C, C, 3), 3 * C, 0.5)
    sd[prefix + "out_layers.3.bias"] = g.bias(C)


def synth_diffusion(cfg: ModelConfig, seed=0):
    """`diffusion_decoder.pth` (DiffusionTts.state_dict(), diffusion_decoder.py:134-220)."""
    g = _Gen(seed * 1000 + 2)
    C, H = cfg.diff_dim, cfg.diff_heads
    cin, cout = cfg.diff_in_channels, cfg.diff_out_channels
    sd = {}
    sd["unconditioned_embedding"] = g.normal((1, C, 1), 1.0)
    sd["inp_block.weight"] = g.lin((C, cin, 3), 3 * cin)
    sd["inp_block.bias"] = g.bias(C)
    for i in (0, 2):
        sd[f"time_embed.{i}.weight"] = g.lin((C, C), C)
        sd[f"time_embed.{i}.bias"] = g.bias(C)
    sd["code_embedding.weight"] = g.normal((cfg.diff_in_tokens, C), 1.0)
    for i in range(3):
        _attention_block(sd, g, f"code_converter.{i}.", C, H, True)
    sd["code_norm.weight"] = g.gamma(C)
    sd["code_norm.bias"] = g.beta(C)
    sd["latent_conditioner.0.weight"] = g.lin((C, cfg.ar_dim, 3), 3 * cfg.ar_dim)
    sd["latent_conditioner.0.bias"] = g.bias(C)
    for i in range(1, 5):
        _attention_block(sd, g, f"latent_conditioner.{i}.", C, H, True)
    sd["contextual_embedder.0.weight"] = g.lin((C, cin, 3), 3 * cin)
    sd["contextual_embedder.0.bias"] = g.bias(C)
    sd["contextual_embedder.1.weight"] = g.lin((2 * C, C, 3), 3 * C)
    sd["contextual_embedder.1.bias"] = g.bias(2 * C)
    for i in range(2, 7):
        _attention_block(sd, g, f"contextual_embedder.{i}.", 2 * C, H, True)
    for i in range(3):
        _diff_resblock(sd, g, f"conditioning_timestep_integrator.{i}.resblk.", C)
        _attention_block(sd, g, f"conditioning_timestep_integrator.{i}.attn.", C, H, True)
    sd["integrating_conv.weight"] = g.lin((C, 2 * C, 1), 2 * C)
    sd["integrating_conv.bias"] = g.bias(C)
    sd["mel_head.weight"] = g.lin((cin, C, 3), 3 * C)
    sd["mel_head.bias"] = g.bias(cin)
    for i in range(cfg.diff_layers):
        _diff_resblock(sd, g, f"layers.{i}.resblk.", C)
        _attention_block(sd, g, f"layers.{i}.attn.", C, H, True)
    for i in range(cfg.diff_layers, cfg.diff_layers + 3):
        _diff_resblock(sd, g, f"layers.{i}.", C)
    sd["out.0.weight"] = g.gamma(C)
    sd["out.0.bias"] = g.beta(C)
    sd["out.2.weight"] = g.lin((cout, C, 3), 3 * C)
    sd["out.2.bias"] = g.bias(cout)
    return sd


def synth_clvp(cfg: ModelConfig, seed=0):
    """`clvp2.pth` (CLVP.state_dict() with use_xformers=True, clvp.py:19-98)."""
    g = _Gen(seed * 1000 + 3)
    D = cfg.clvp_dim
    sd = {}
    sd["temperature"] = torch.tensor(1.0)
    sd["text_emb.weight"] = g.normal((cfg.clvp_text_tokens, D), 1.0)
    sd["to_text_latent.weight"] = g.lin((D, D), D)
    sd["speech_emb.weight"] = g.normal((cfg.clvp_speech_tokens, D), 1.0)
    sd["to_speech_latent.weight"] = g.lin((D, D), D)
    for enc in ("text", "speech"):
        p = f"{enc}_transformer.transformer."
        for l in range(cfg.clvp_depth):
            a = f"{p}attn_layers.layers.{2 * l}."
            sd[a + "0.0.g"] = g.gamma(D)
            for nm in ("to_q", "to_k", "to_v"):
                sd[a + f"1.wrap.{nm}.weight"] = g.lin((D, D), D)
            sd[a + "1.wrap.to_out.weight"] = g.lin((D, D), D, 0.5)
            sd[a + "1.wrap.to_out.bias"] = g.bias(D)
            f = f"{p}attn_layers.layers.{2 * l + 1}."
            sd[f + "0.0.g"] = g.gamma(D)
            sd[f + "1.wrap.net.0.proj.weight"] = g.lin((4 * D, D), D)
            sd[f + "1.wrap.net.0.proj.bias"] = g.bias(4 * D)
            sd[f + "1.wrap.net.3.weight"] = g.lin((D, 2 * D), 2 * D, 0.5)
            sd[f + "1.wrap.net.3.bias"] = g.bias(D)
        sd[p + "attn_layers.rotary_pos_emb.inv_freq"] = 1.0 / (10000 ** (torch.arange(0, 32, 2).float() / 32))
        sd[p + "norm.weight"] = g.gamma(D)
        sd[p + "norm.bias"] = g.beta(D)
    return sd


def synth_cvvp(cfg: ModelConfig, seed=0):
    """`cvvp.pth` (CVVP.state_dict() as api.py:254-255 builds it: mel_codes=8192, depths 8, latent_multiplier 1;
    cvvp.py:64-106). The transformers are plain ContinuousTransformerWrappers: no `.wrap.` in the layer keys."""
    g = _Gen(seed * 1000 + 6)
    D = cfg.cvvp_dim
    sd = {}
    sd["temperature"] = torch.tensor(1.0)
    sd["cond_emb.0.weight"] = g.lin((D // 2, 80, 5), 80 * 5)
    sd["cond_emb.0.bias"] = g.bias(D // 2)
    sd["cond_emb.1.weight"] = g.lin((D, D // 2, 3), (D // 2) * 3)
    sd["cond_emb.1.bias"] = g.bias(D)
    sd["to_conditioning_latent.weight"] = g.lin((D, D), D)
    sd["speech_emb.emb.weight"] = g.normal((cfg.clvp_speech_tokens, D), 1.0)
    sd["to_speech_latent.weight"] = g.lin((D, D), D)
    for enc in ("conditioning", "speech"):
        p = f"{enc}_transformer.transformer."
        for l in range(cfg.cvvp_depth):
            a = f"{p}attn_layers.layers.{2 * l}."
            sd[a + "0.0.g"] = g.gamma(D)
            for nm in ("to_q", "to_k", "to_v"):
                sd[a + f"1.{nm}.weight"] = g.lin((D, D), D)
            sd[a + "1.to_out.weight"] = g.lin((D, D), D, 0.5)
            sd[a + "1.to_out.bias"] = g.bias(D)
            f = f"{p}attn_layers.layers.{2 * l + 1}."
            sd[f + "0.0.g"] = g.gamma(D)
            sd[f + "1.net.0.proj.weight"] = g.lin((2 * D, D), D)          # ff_mult = 1, GLU: 2 x inner rows
            sd[f + "1.net.0.proj.bias"] = g.bias(2 * D)
            sd[f + "1.net.3.weight"] = g.lin((D, D), D, 0.5)
            sd[f + "1.net.3.bias"] = g.bias(D)
        sd[p + "attn_layers.rotary_pos_emb.inv_freq"] = 1.0 / (10000 ** (torch.arange(0, 32, 2).float() / 32))
        sd[p + "norm.weight"] = g.gamma(D)
        sd[p + "norm.bias"] = g.beta(D)
        c = f"{enc}_transformer.pre_combiner."
        sd[c + "0.weight"] = g.lin((D, D, 1), D)
        sd[c + "0.bias"] = g.bias(D)
        _attention_block(sd, g, c + "1.", D, cfg.cvvp_heads, rel_pos=False)
        sd[c + "2.weight"] = g.lin((D, D, 1), D)
        sd[c + "2.bias"] = g.bias(D)
    return sd


def _wn(sd, g, prefix, shape, fan_in, gain=1.0):
    """weight-norm pair (weight_g over all dims but 0, vocoder.py:290-298)."""
    v = g.lin(shape, fan_in, gain)
    norm = v.reshape(shape[0], -1).norm(dim=1).reshape(shape[0], *([1] * (len(shape) - 1)))
    sd[prefix + "bias"] = g.bias(shape[0] if "convt" not in prefix else shape[1])
    sd[prefix + "weight_g"] = norm * (1.0 + g.normal(norm.shape, 0.05))
    sd[prefix + "weight_v"] = v


def synth_vocoder(cfg: ModelConfig, seed=0):
    """`vocoder.pth['model_g']` (UnivNetGenerator.state_dict() before remove_weight_norm)."""
    g = _Gen(seed * 1000 + 4)
    ch, nz, mel, hid = cfg.voc_channels, cfg.voc_noise_dim, cfg.voc_mel, cfg.voc_kp_hidden
    nl = len(VOC_DILATIONS)
    sd = {}
    for b, s in enumerate(VOC_STRIDES):
        p = f"res_stack.{b}."
        kp = p + "kernel_predictor."
        _wn(sd, g, kp + "input_conv.0.", (hid, mel, 5), 5 * mel)
        for r in range(3):
            _wn(sd, g, kp + f"residual_convs.{r}.1.", (hid, hid, 3), 3 * hid)
            _wn(sd, g, kp + f"residual_convs.{r}.3.", (hid, hid, 3), 3 * hid, 0.5)
        # LVC kernels of scale ~1/sqrt(fan_in of the LVC = 3*ch) keep the gated residual bounded
        _wn(sd, g, kp + "kernel_conv.", (ch * 2 * ch * 3 * nl, hid, 3), 3 * hid, 1.0 / math.sqrt(3 * ch))
        _wn(sd, g, kp + "bias_conv.", (2 * ch * nl, hid, 3), 3 * hid, 0.1)
        _wn(sd, g, p + "convt_pre.1.", (ch, ch, 2 * s), 2 * ch)          # ConvTranspose1d: [in, out, k]
        for d in range(nl):
            _wn(sd, g, p + f"conv_blocks.{d}.1.", (ch, ch, 3), 3 * ch)
    _wn(sd, g, "conv_pre.", (ch, nz, 7), 7 * nz)
    _wn(sd, g, "conv_post.1.", (1, ch, 7), 7 * ch)
    return sd


def synth_hifigan(cfg: ModelConfig, seed=0):
    """`hifidecoder.pth` (HifiganGenerator.state_dict() as api_fast.py:221-227 builds it, weight norm in place:
    hifigan_decoder.py:159-238)."""
    from .config import HIFI_UP_FACTORS, HIFI_RES_KERNELS
    g = _Gen(seed * 1000 + 7)
    C0, Cin = cfg.hifi_channels, cfg.ar_dim
    sd = {}

    def wn(prefix, shape, fan_in, nbias, gain=1.0):
        v = g.lin(shape, fan_in, gain)
        norm = v.reshape(shape[0], -1).norm(dim=1).reshape(shape[0], *([1] * (len(shape) - 1)))
        sd[prefix + "bias"] = g.bias(nbias)
        sd[prefix + "weight_g"] = norm * (1.0 + g.normal(norm.shape, 0.05))
        sd[prefix + "weight_v"] = v

    wn("conv_pre.", (C0, Cin, 7), 7 * Cin, C0)
    ch = C0
    for i, u in enumerate(HIFI_UP_FACTORS):
        # ConvTranspose1d weight [in, out, k]: every output sums in * 2 taps
        wn(f"ups.{i}.", (ch, ch // 2, 2 * u), 2 * ch, ch // 2)
        ch //= 2
        for j, k in enumerate(HIFI_RES_KERNELS):
            p = f"resblocks.{i * len(HIFI_RES_KERNELS) + j}."
            for m in range(3):
                wn(p + f"convs1.{m}.", (ch, ch, k), k * ch, ch)
                wn(p + f"convs2.{m}.", (ch, ch, k), k * ch, ch, 0.5)
    wn("conv_post.", (1, ch, 7), 7 * ch, 1, 3.0)
    sd["cond_layer.weight"] = g.lin((C0, Cin, 1), Cin)
    sd["cond_layer.bias"] = g.bias(C0)
    return sd


def synth_rlg(C, seed=0):
    """`rlg_auto.pth` / `rlg_diffuser.pth` (RandomLatentConverter, random_latent_generator.py:40-50)."""
    g = _Gen(seed * 1000 + 5 + C)
    sd = {}
    for i in range(5):
        sd[f"layers.{i}.weight"] = g.normal((C, C), 1.0 / 0.1)     # EqualLinear: randn / lr_mul
        sd[f"layers.{i}.bias"] = torch.zeros(C)
    sd["layers.5.weight"] = g.lin((C, C), C)
    sd["layers.5.bias"] = g.bias(C)
    return sd


W2V_VOCAB = ["<pad>", "<s>", "</s>", "<unk>", "|"] + list("'abcdefghijklmnopqrstuvwxyz,.!?-")


def wav2vec_config(size="full"):
    """HF Wav2Vec2Config fields of the redaction aligner: "full" = wav2vec2-large-robust (24 x 1024, 16 heads, FF 4096),
    "small" = the same architecture at 2 x 256 (tests)."""
    full = size == "full"
    H = 1024 if full else 256
    return {
        "model_type": "wav2vec2", "architectures": ["Wav2Vec2ForCTC"],
        "do_stable_layer_norm": True, "feat_extract_norm": "layer", "conv_bias": True,
        "feat_extract_activation": "gelu", "hidden_act": "gelu",
        "conv_dim": [512 if full else 256] * 7, "conv_kernel": [10, 3, 3, 3, 3, 2, 2], "conv_stride": [5, 2, 2, 2, 2, 2, 2],
        "hidden_size": H, "num_attention_heads": H // 64, "intermediate_size": 4 * H,
        "num_hidden_layers": 24 if full else 2,
        "num_conv_pos_embeddings": 128 if full else 32, "num_conv_pos_embedding_groups": 16 if full else 4,
        "layer_norm_eps": 1e-5, "vocab_size": len(W2V_VOCAB), "pad_token_id": 0,
        "hidden_dropout": 0.0, "attention_dropout": 0.0, "activation_dropout": 0.0, "feat_proj_dropout": 0.0,
        "final_dropout": 0.0, "layerdrop": 0.0, "mask_time_prob": 0.0,
    }


def synth_wav2vec(cfg="small", seed=0):
    """Seeded Wav2Vec2ForCTC checkpoint for the redaction aligner: (config dict, state dict in the HF key layout,
    character vocab {token: id}). `cfg`: "small", "full" or a config dict (wav2vec_config). The positional conv's weight
    norm is stored in the `parametrizations.weight.original0/1` form. Not part of synth_all."""
    if isinstance(cfg, str):
        cfg = wav2vec_config(cfg)
    g = _Gen(seed * 1000 + 9)
    C, H, FF = cfg["conv_dim"][0], cfg["hidden_size"], cfg["intermediate_size"]
    V, k, G = cfg["vocab_size"], cfg["num_conv_pos_embeddings"], cfg["num_conv_pos_embedding_groups"]
    sd = {}
    p = "wav2vec2."
    cin = 1
    for i, kk in enumerate(cfg["conv_kernel"]):
        q = p + f"feature_extractor.conv_layers.{i}."
        sd[q + "conv.weight"] = g.lin((C, cin, kk), cin * kk)
        sd[q + "conv.bias"] = g.bias(C)
        sd[q + "layer_norm.weight"] = g.gamma(C)
        sd[q + "layer_norm.bias"] = g.beta(C)
        cin = C
    q = p + "feature_projection."
    sd[q + "layer_norm.weight"], sd[q + "layer_norm.bias"] = g.gamma(C), g.beta(C)
    sd[q + "projection.weight"], sd[q + "projection.bias"] = g.lin((H, C), C), g.bias(H)
    q = p + "encoder.pos_conv_embed.conv."
    v = g.lin((H, H // G, k), k * H // G, 0.5)
    norm = v.permute(2, 0, 1).reshape(k, -1).norm(dim=1).reshape(1, 1, k)
    sd[q + "bias"] = g.bias(H)
    sd[q + "parametrizations.weight.original0"] = norm * (1.0 + g.normal(norm.shape, 0.05))
    sd[q + "parametrizations.weight.original1"] = v
    sd[p + "encoder.layer_norm.weight"], sd[p + "encoder.layer_norm.bias"] = g.gamma(H), g.beta(H)
    for l in range(cfg["num_hidden_layers"]):
        q = p + f"encoder.layers.{l}."
        for n in ("q", "k", "v", "out"):
            sd[q + f"attention.{n}_proj.weight"] = g.lin((H, H), H)
            sd[q + f"attention.{n}_proj.bias"] = g.bias(H)
        sd[q + "layer_norm.weight"], sd[q + "layer_norm.bias"] = g.gamma(H), g.beta(H)
        sd[q + "final_layer_norm.weight"], sd[q + "final_layer_norm.bias"] = g.gamma(H), g.beta(H)
        sd[q + "feed_forward.intermediate_dense.weight"] = g.lin((FF, H), H)
        sd[q + "feed_forward.intermediate_dense.bias"] = g.bias(FF)
        sd[q + "feed_forward.output_dense.weight"] = g.lin((H, FF), FF, 0.5)
        sd[q + "feed_forward.output_dense.bias"] = g.bias(H)
    sd["lm_head.weight"], sd["lm_head.bias"] = g.lin((V, H), H, 2.0), g.bias(V, 0.5)
    vocab = {t: i for i, t in enumerate(W2V_VOCAB[:V])}
    return cfg, sd, vocab


def synth_all(cfg: ModelConfig, seed=0, suppress_stop=True):
    return {
        "autoregressive": synth_autoregressive(cfg, seed, suppress_stop),
        "diffusion": synth_diffusion(cfg, seed),
        "clvp": synth_clvp(cfg, seed),
        "vocoder": synth_vocoder(cfg, seed),
        "rlg_auto": synth_rlg(cfg.ar_dim, seed),
        "rlg_diffuser": synth_rlg(2 * cfg.diff_dim, seed + 1),
        "cvvp": synth_cvvp(cfg, seed),
        "hifigan": synth_hifigan(cfg, seed),
    }


def write_models_dir(path, cfg: ModelConfig, seed=0, suppress_stop=True):
    """Write a models_dir the reference `TextToSpeech(models_dir=...)` layout expects (api.py:31-40)."""
    os.makedirs(path, exist_ok=True)
    sds = synth_all(cfg, seed, suppress_stop)
    torch.save(sds["autoregressive"], os.path.join(path, "autoregressive.pth"))
    torch.save(sds["diffusion"], os.path.join(path, "diffusion_decoder.pth"))
    torch.save(sds["clvp"], os.path.join(path, "clvp2.pth"))
    torch.save({"model_g": sds["vocoder"]}, os.path.join(path, "vocoder.pth"))
    torch.save(synth_rlg(cfg.ar_dim, seed), os.path.join(path, "rlg_auto.pth"))
    torch.save(synth_rlg(2 * cfg.diff_dim, seed), os.path.join(path, "rlg_diffuser.pth"))
    torch.save(sds["cvvp"], os.path.join(path, "cvvp.pth"))
    torch.save(sds["hifigan"], os.path.join(path, "hifidecoder.pth"))
    return sds
