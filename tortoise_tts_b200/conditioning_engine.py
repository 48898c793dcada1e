"""Conditioning front-end on the sm_90a kernels (SURVEY §8f-1): reference clips -> (auto latent [1, D], diffusion latent
[1, 2C]).

Mirrors `TextToSpeech.get_conditioning_latents` (tortoise/api.py:258-299):
  * AR latent: format_conditioning (api.py:73-84) -> TorchMelSpectrogram (models/arch_util.py:295-331) ->
    ConditioningEncoder (models/autoregressive.py:204-228) -> position 0 -> mean over clips (autoregressive.py:444-452)
  * diffusion latent: resample 22.05 -> 24 kHz (api.py:284), pad/truncate to 102400, TacotronSTFT mel (utils/audio.py:
    151-191, utils/stft.py:94-157) -> contextual_embedder (models/diffusion_decoder.py:186-192) -> mean over positions
    of all clips (diffusion_decoder.py:222-230)
and `get_random_conditioning_latents` (api.py:301-309, models/random_latent_generator.py:8-50).

Host side builds the constant tables (window, DFT twiddles, mel filterbanks, resampling kernels) in float64 the way
torchaudio / librosa build them; every per-sample arithmetic operation runs in libttb.so.
"""
import math
import random

import numpy as np
import torch

from . import lib
from .config import ModelConfig
from .diffusion_engine import _AttnW, _bf, _f, _groups_for, _pad_k

COND_LENGTH = 132300        # api.py:73
DIFF_COND_LENGTH = 102400   # api.py:285
N_FFT, HOP = 1024, 256


def _mel_filterbank(sr, n_fft, n_mels, fmin, fmax, mel_scale):
    """Triangular mel filters with Slaney area normalisation, float64 [n_mels, n_fft//2+1].
    'htk': torchaudio melscale_fbanks defaults used by TorchMelSpectrogram (arch_util.py:307-311, norm='slaney');
    'slaney': librosa.filters.mel defaults used by TacotronSTFT (utils/audio.py:158-160)."""
    if mel_scale == "htk":
        def to_mel(f):
            return 2595.0 * np.log10(1.0 + np.asarray(f, dtype=np.float64) / 700.0)

        def to_hz(m):
            return 700.0 * (10.0 ** (np.asarray(m, dtype=np.float64) / 2595.0) - 1.0)
    else:
        f_sp, min_log_hz, logstep = 200.0 / 3, 1000.0, math.log(6.4) / 27.0
        min_log_mel = min_log_hz / f_sp

        def to_mel(f):
            f = np.asarray(f, dtype=np.float64)
            return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-10) / min_log_hz) / logstep, f / f_sp)

        def to_hz(m):
            m = np.asarray(m, dtype=np.float64)
            return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)
    freqs = np.linspace(0.0, sr / 2.0, n_fft // 2 + 1)
    pts = to_hz(np.linspace(to_mel(fmin), to_mel(fmax), n_mels + 2))
    fdiff = np.diff(pts)
    ramps = pts[:, None] - freqs[None, :]
    w = np.maximum(0.0, np.minimum(-ramps[:-2] / fdiff[:-1, None], ramps[2:] / fdiff[1:, None]))
    return w * (2.0 / (pts[2:n_mels + 2] - pts[:n_mels]))[:, None]


def _resample_kernels(orig, new, lowpass_filter_width=6, rolloff=0.99):
    """torchaudio.functional.resample's windowed-sinc polyphase bank (sinc_interp_hann). Returns (kernels float32
    [new/g, klen], orig/g, new/g, width). torchaudio evaluates this table in the waveform's dtype (float32)."""
    g = math.gcd(orig, new)
    o, n = orig // g, new // g
    base = min(o, n) * rolloff
    width = math.ceil(lowpass_filter_width * o / base)
    idx = torch.arange(-width, width + o, dtype=torch.float32)[None, :] / o
    t = torch.arange(0, -n, -1, dtype=torch.float32)[:, None] / n + idx
    t = (t * base).clamp_(-lowpass_filter_width, lowpass_filter_width)
    window = torch.cos(t * math.pi / lowpass_filter_width / 2) ** 2
    t = t * math.pi
    k = torch.where(t == 0, torch.tensor(1.0), t.sin() / t) * window * (base / o)
    return k.contiguous(), o, n, width


class ConditioningEngine:
    def __init__(self, sd_ar, sd_diff, cfg: ModelConfig, device="cuda", mel_norms=None):
        self.cfg = cfg
        self.dev = torch.device(device)
        dev = self.dev
        D, C, H = cfg.ar_dim, cfg.diff_dim, cfg.diff_heads
        self.D, self.C2 = D, 2 * C
        # --- tables
        n = np.arange(N_FFT)
        self.window = torch.from_numpy(0.5 - 0.5 * np.cos(2.0 * np.pi * n / N_FFT)).float().to(dev)   # periodic hann
        tw = np.stack([np.cos(2.0 * np.pi * n / N_FFT), np.sin(2.0 * np.pi * n / N_FFT)], axis=1)
        self.twiddle = torch.from_numpy(tw).float().contiguous().to(dev)
        self.fb_ar = torch.from_numpy(_mel_filterbank(22050, N_FFT, 80, 0.0, 8000.0, "htk")).float().contiguous().to(dev)
        self.fb_diff = torch.from_numpy(_mel_filterbank(24000, N_FFT, 100, 0.0, 12000.0, "slaney")).float().contiguous().to(dev)
        k, self.rs_down, self.rs_up, self.rs_width = _resample_kernels(22050, 24000)
        self.rs_kernels = k.to(dev)
        if mel_norms is None:
            raise ValueError("mel_norms (reference asset tortoise/data/mel_norms.pth, 80 floats) is required")
        self.mel_norms = _f(mel_norms.reshape(-1), dev)
        # --- AR conditioning encoder (autoregressive.py:204-228)
        self.kpad_ar = 128
        self.w_init = _bf(_pad_k(sd_ar["conditioning_encoder.init.weight"], self.kpad_ar), dev)
        self.b_init = _f(sd_ar["conditioning_encoder.init.bias"], dev)
        self.ar_attn = [_AttnW(sd_ar, f"conditioning_encoder.attn.{i}.", D, cfg.ar_heads, dev) for i in range(cfg.cond_enc_blocks)]
        self.ar_heads, self.diff_heads = cfg.ar_heads, H
        if sd_diff is None:       # api_fast needs the autoregressive conditioning latent only (api_fast.py:225-246)
            return
        # --- diffusion contextual embedder (diffusion_decoder.py:186-192)
        self.kpad_diff = 128
        self.w_c0 = _bf(_pad_k(sd_diff["contextual_embedder.0.weight"], self.kpad_diff), dev)
        self.b_c0 = _f(sd_diff["contextual_embedder.0.bias"], dev)
        self.w_c1 = _bf(sd_diff["contextual_embedder.1.weight"].permute(0, 2, 1).reshape(2 * C, 3 * C), dev)
        self.b_c1 = _f(sd_diff["contextual_embedder.1.bias"], dev)
        self.ctx_attn = [_AttnW(sd_diff, f"contextual_embedder.{i}.", 2 * C, H, dev) for i in range(2, 7)]
        self.ar_heads, self.diff_heads = cfg.ar_heads, H

    # ------------------------------------------------------------------ AttentionBlock on x fp32 [T, C] (in place)
    def _attn_block(self, aw, x, T, C, H):
        dev = self.dev
        groups = _groups_for(C)
        ch = C // H
        a = torch.empty(T, C, dtype=torch.bfloat16, device=dev)
        qkv = torch.empty(T, 3 * C, dtype=torch.bfloat16, device=dev)
        o = torch.empty(T, C, dtype=torch.bfloat16, device=dev)
        part = lib.groupnorm_scratch(1, groups, dev)
        lib.groupnorm(x, 1, T, C, groups, aw.gn_g, aw.gn_b, part, out_bf16=a, ldo=C)
        lib.gemm(a, aw.wqkv, M=T, N=3 * C, K=C, bias=aw.bqkv, out_bf16=qkv)
        # QKVAttentionLegacy scales q and k by ch^-1/4 each (arch_util.py:64-67)
        lib.attention(qkv, o, nseq=1, T=T, H=H, ld=3 * C, ldo=C, k_off=C, v_off=2 * C, scale=1.0 / math.sqrt(ch),
                      bias=aw.table(T), bias_sat=64 if aw.rel_emb is not None else 0, head_dim=0 if ch == 64 else ch)
        lib.gemm(o, aw.wproj, M=T, N=C, K=C, bias=aw.bproj, residual=x, out_f32=x)

    # ------------------------------------------------------------------ mel front ends
    def ar_mel(self, clip, out_f32=None):
        """clip fp32 [COND_LENGTH] on the device -> bf16 token-major [frames, 128] (80 mels + zero padding)."""
        n = clip.numel()
        frames = 1 + n // HOP
        out = torch.empty(frames, self.kpad_ar, dtype=torch.bfloat16, device=self.dev)
        lib.audio_stft_mel(clip, n, N_FFT, HOP, self.window, self.twiddle, self.fb_ar, 80, 2, False, 1e-5, self.mel_norms,
                           out_bf16=out, ldo=self.kpad_ar, out_f32=out_f32)
        return out, frames

    def diffusion_mel(self, clip22, out_f32=None):
        """clip fp32 [n] at 22.05 kHz -> resample to 24 kHz, pad / truncate to 102400 -> bf16 [401, 128] (100 mels)."""
        n = clip22.numel()
        m = min(DIFF_COND_LENGTH, int(math.ceil(self.rs_up * n / self.rs_down)))
        wav = torch.zeros(DIFF_COND_LENGTH, dtype=torch.float32, device=self.dev)
        lib.audio_resample(clip22, n, self.rs_kernels, self.rs_down, self.rs_up, self.rs_kernels.shape[1], self.rs_width, wav, m)
        frames = 1 + DIFF_COND_LENGTH // HOP
        out = torch.empty(frames, self.kpad_diff, dtype=torch.bfloat16, device=self.dev)
        lib.audio_stft_mel(wav, DIFF_COND_LENGTH, N_FFT, HOP, self.window, self.twiddle, self.fb_diff, 100, 1, True, 1e-5,
                           None, out_bf16=out, ldo=self.kpad_diff, out_f32=out_f32)
        return out, frames

    @staticmethod
    def format_clip(clip, start=None):
        """format_conditioning's pad / random crop (api.py:77-82). clip [1, n] or [n]; returns 1-D [COND_LENGTH]."""
        clip = clip.reshape(-1)
        gap = clip.shape[-1] - COND_LENGTH
        if gap < 0:
            return torch.nn.functional.pad(clip, (0, -gap))
        if gap > 0:
            s = random.randint(0, gap) if start is None else int(start)
            return clip[s:s + COND_LENGTH]
        return clip

    # ------------------------------------------------------------------ latents
    def ar_latent(self, clips, starts=None, return_mels=False):
        dev, D = self.dev, self.D
        out = torch.empty(D, dtype=torch.float32, device=dev)
        mels = []
        for i, c in enumerate(clips):
            w = self.format_clip(c.to(dev).float(), None if starts is None else starts[i]).contiguous()
            mf = torch.empty(80, 1 + COND_LENGTH // HOP, dtype=torch.float32, device=dev) if return_mels else None
            mel, T = self.ar_mel(w, mf)
            if return_mels:
                mels.append(mf.unsqueeze(0))
            x = torch.empty(T, D, dtype=torch.float32, device=dev)
            lib.gemm(mel, self.w_init, M=T, N=D, K=self.kpad_ar, bias=self.b_init, out_f32=x)
            for aw in self.ar_attn:
                self._attn_block(aw, x, T, D, self.ar_heads)
            lib.mean_rows(x, 1, D, D, 1.0 / len(clips), out, accumulate=i > 0)      # h[:, :, 0], mean over clips
        lat = out.reshape(1, D)
        return (lat, torch.stack(mels, dim=1)) if return_mels else lat

    def diffusion_latent(self, clips, return_mels=False):
        dev, C2 = self.dev, self.C2
        C = C2 // 2
        out = torch.empty(C2, dtype=torch.float32, device=dev)
        mels = []
        T2 = None
        per_clip = []
        for c in clips:
            mf = torch.empty(100, 1 + DIFF_COND_LENGTH // HOP, dtype=torch.float32, device=dev) if return_mels else None
            mel, T0 = self.diffusion_mel(c.to(dev).float().reshape(-1).contiguous(), mf)
            if return_mels:
                mels.append(mf.unsqueeze(0))
            # conv k=3, stride 2, padding 1 = every second row of the stride-1 convolution
            y0 = torch.empty(T0, C, dtype=torch.float32, device=dev)
            lib.gemm(mel, self.w_c0, M=T0, N=C, K=self.kpad_diff, taps=3, pad=1, bias=self.b_c0, out_f32=y0)
            T1 = (T0 + 1) // 2
            a1 = torch.empty(T1, C, dtype=torch.bfloat16, device=dev)
            lib.cast_pad_bf16(y0, T1, C, 2 * C, a1, C)                               # rows 0, 2, 4, ...
            y1 = torch.empty(T1, C2, dtype=torch.float32, device=dev)
            lib.gemm(a1, self.w_c1, M=T1, N=C2, K=C, taps=3, pad=1, bias=self.b_c1, out_f32=y1)
            T2 = (T1 + 1) // 2
            x = y1[0::2].contiguous()
            for aw in self.ctx_attn:
                self._attn_block(aw, x, T2, C2, self.diff_heads)
            per_clip.append((x, T2))
        total = sum(t for _, t in per_clip)
        for i, (x, t) in enumerate(per_clip):
            lib.mean_rows(x, t, C2, C2, 1.0 / total, out, accumulate=i > 0)          # cat over time, mean over time
        lat = out.reshape(1, C2)
        return (lat, torch.stack(mels, dim=1)) if return_mels else lat


class RandomLatentEngine:
    """RandomLatentConverter (random_latent_generator.py:40-50): 5 x EqualLinear(lr_mul 0.1) + Linear on a normal draw.
    The draw itself comes from torch's CPU generator, as in the reference (`torch.randn(ref.shape[0], C)` on the CPU)."""

    def __init__(self, sd, C, device="cuda"):
        self.C, self.dev = C, torch.device(device)
        self.w = [_f(sd[f"layers.{i}.weight"], self.dev) for i in range(6)]
        self.b = [_f(sd[f"layers.{i}.bias"], self.dev) for i in range(6)]

    def __call__(self, r=None):
        C, dev = self.C, self.dev
        r = torch.randn(1, C) if r is None else r
        x = r.reshape(-1).to(device=dev, dtype=torch.float32).contiguous()
        for i in range(5):
            y = torch.empty(C, dtype=torch.float32, device=dev)
            lib.equal_linear(x, C, self.w[i], self.b[i], C, y, wscale=(1 / math.sqrt(C)) * 0.1, bscale=0.1, slope=0.2,
                             gain=2 ** 0.5)
            x = y
        y = torch.empty(C, dtype=torch.float32, device=dev)
        lib.equal_linear(x, C, self.w[5], self.b[5], C, y)
        return y.reshape(1, C)
