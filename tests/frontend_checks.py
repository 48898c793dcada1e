"""Float64 restatements of the conditioning front-end and the small helper kernels, the per-element bounds their fp32
forms must meet, and the cases that run a kernel against them between NaN canaries.

Every case takes `L`, a module with the signatures of tortoise_tts_b200.lib, and a device. The GPU tests
(test_gpu_frontend_kernels.py) pass the library itself. test_frontend_checks_host.py passes the fp32 torch emulation of
tests/lib_emu.py, which must pass, and subtly wrong versions of it, which must be rejected: each bound is shown to
catch the mistakes it is there for.

Bounds (u = 2^-24, the fp32 unit roundoff). An fp32 sum of n terms is off from the exact sum by at most
c * n * u * sum|terms|; c = 4 also covers the fast-math intrinsics (`--use_fast_math`: approximate division, sqrt, log,
with errors of a few ulp). Each bound is carried through the later operations of the kernel with the magnitudes of the
float64 result, and is stated where it is computed. The reference reads the same fp32 tables as the kernel (window,
twiddles, filterbanks, resampling bank from conditioning_engine, pinned by test_oracle_conditioning.py), so a case checks
the kernel and not the table construction.
"""
import json
import math
import os

import numpy as np
import torch

U = 2.0 ** -24
CF = 4.0                     # the c of c * n * u * sum|terms|
BF16_REL = 2.0 ** -8         # round-to-nearest bf16 (8 significant bits): |bf16(v) - v| <= 2^-8 |v|
NAN = float("nan")
FLOOR = 1e-5

_MEL_NORMS = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tortoise_tts_b200", "data",
                          "mel_norms.json")

# the two production configurations of ttb_audio_stft_mel (conditioning_engine.ar_mel / diffusion_mel)
STFT_CONFIGS = {
    "ar": dict(n_mels=80, power=2, clip=False, div=True, prod_n=132300),
    "diffusion": dict(n_mels=100, power=1, clip=True, div=False, prod_n=102400),
}
STFT_SIGNALS = ("zeros", "impulse0", "impulse1", "impulse_n2", "impulse_n1", "burst", "dc", "loud", "noise")
RESAMPLE_RATIOS = ((22050, 24000), (24000, 16000))


def within(name, got, want, bound):
    """Every element of `got` is finite (a NaN canary left in place means an element was not written) and within its
    bound of `want`. Returns the largest error relative to its bound."""
    g = got.detach().double().cpu().numpy() if torch.is_tensor(got) else np.asarray(got, dtype=np.float64)
    want = np.broadcast_to(np.asarray(want, dtype=np.float64), g.shape)
    bound = np.broadcast_to(np.asarray(bound, dtype=np.float64), g.shape)
    bad = ~np.isfinite(g)
    assert not bad.any(), "%s: %d elements not written or not finite, first at %s" % (
        name, int(bad.sum()), np.argwhere(bad)[0].tolist())
    err = np.abs(g - want)
    ratio = np.divide(err, bound, out=np.where(err > 0, np.inf, 0.0), where=bound > 0)     # a zero bound means exact
    worst = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
    assert ratio[worst] <= 1.0, "%s: error %.3e > bound %.3e at %s (got %r, want %r)" % (
        name, err[worst], bound[worst], list(worst), g[worst], want[worst])
    return float(ratio[worst])


def untouched(name, t):
    assert torch.isnan(t.float()).all(), "%s: canary overwritten (%d elements)" % (name, int((~torch.isnan(t.float())).sum()))


def _f64(t):
    return t.detach().double().cpu().numpy()


# ------------------------------------------------------------------ tables
class Tables:
    """The fp32 tables the conditioning engine feeds the front-end kernels, on `dev`."""

    def __init__(self, dev):
        from tortoise_tts_b200.conditioning_engine import HOP, N_FFT, _mel_filterbank, _resample_kernels
        self.n_fft, self.hop = N_FFT, HOP
        n = np.arange(N_FFT)
        # the expressions of ConditioningEngine.__init__
        self.window = torch.from_numpy(0.5 - 0.5 * np.cos(2.0 * np.pi * n / N_FFT)).float().to(dev)
        tw = np.stack([np.cos(2.0 * np.pi * n / N_FFT), np.sin(2.0 * np.pi * n / N_FFT)], axis=1)
        self.twiddle = torch.from_numpy(tw).float().contiguous().to(dev)
        self.fb = {"ar": torch.from_numpy(_mel_filterbank(22050, N_FFT, 80, 0.0, 8000.0, "htk")).float().contiguous().to(dev),
                   "diffusion": torch.from_numpy(_mel_filterbank(24000, N_FFT, 100, 0.0, 12000.0, "slaney")).float()
                   .contiguous().to(dev)}
        with open(_MEL_NORMS) as f:
            self.mel_norms = torch.tensor(json.load(f)["mel_norms"], dtype=torch.float32).to(dev)
        self.resample = {r: _resample_kernels(*r) for r in RESAMPLE_RATIOS}
        self.resample = {r: (k.to(dev), d, up, w) for r, (k, d, up, w) in self.resample.items()}


# ------------------------------------------------------------------ STFT -> mel -> log
def stft_signal(kind, n, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.zeros(n)
    if kind.startswith("impulse"):
        x[{"impulse0": 0, "impulse1": 1, "impulse_n2": n - 2, "impulse_n1": n - 1}[kind]] = 1.0
    elif kind == "burst":
        a, b = max(0, n // 2 - 150), min(n, n // 2 + 150)
        x[a:b] = torch.rand(b - a, generator=g) * 2 - 1
    elif kind == "dc":
        x[:] = 0.3
    elif kind == "loud":
        x = torch.rand(n, generator=g) * 6 - 3                  # up to +-3: TacotronSTFT clips, TorchMelSpectrogram does not
    elif kind == "noise":
        x = torch.rand(n, generator=g) * 2 - 1
    else:
        assert kind == "zeros", kind
    return x.float()


_DFT = {}


def _dft_tables(twiddle):
    """cos / -sin matrices [n_fft/2+1, n_fft] of the fp32 twiddles, indexed (k * i) mod n_fft as the kernel reads them."""
    tw = _f64(twiddle)
    key = tw.tobytes()
    if key not in _DFT:
        n_fft = tw.shape[0]
        idx = (np.arange(n_fft // 2 + 1)[:, None] * np.arange(n_fft)[None, :]) % n_fft
        _DFT.clear()
        _DFT[key] = (tw[idx, 0], -tw[idx, 1])
    return _DFT[key]


def stft_mel64(x, n_fft, hop, window, twiddle, fb, power, clip, floor_v, div):
    """y = log(max(mel, floor)) [/ div] in float64 on the fp32 inputs, [frames, n_mels], and its per-element bound.

    - frame t covers padded samples [t*hop, t*hop + n_fft) of x reflect-padded by n_fft/2 on both sides (center=True);
      the windowed sample fr = clip(x) * w is exact in float64 (two 24-bit significands).
    - re, im: sums of n_fft products fr * twiddle, each rounded once (the window product and the FMA):
      E_re = c (n_fft + 2) u sum|fr * cos|, E_im likewise with sin.
    - p = re^2 + im^2: E_p = 2|re| E_re + 2|im| E_im + E_re^2 + E_im^2 + c u p. Power 1 takes sqrt(p), whose error is at
      most min(E_p / sqrt(p), sqrt(E_p)) (|sqrt a - sqrt b| = |a - b| / (sqrt a + sqrt b) <= sqrt|a - b|), plus c u sqrt(p).
    - mel = sum_k fb[c, k] spec[k] over n_fft/2 + 1 terms, fb >= 0: E_mel = fb @ E_spec + c (n_fft/2 + 2) u mel.
    - log(max(., floor)) is Lipschitz with constant 1 / max(min, floor): E_y = E_mel / max(mel - E_mel, floor), plus the
      fast-math logf (2^-21.4 absolute near 1, 3 ulp elsewhere): c (2^-23 + 2 u |y|).
    - / div: E_out = E_y / |div| + 2 c u |y / div| (approximate division)."""
    x = _f64(x)
    n = x.shape[0]
    if clip:
        x = np.clip(x, -1.0, 1.0)
    pad = n_fft // 2
    xp = np.pad(x, pad, mode="reflect")
    frames = 1 + n // hop
    fr = xp[np.arange(frames)[:, None] * hop + np.arange(n_fft)[None, :]] * _f64(window)[None, :]
    cm, sm = _dft_tables(twiddle)
    re, im = fr @ cm.T, fr @ sm.T
    afr = np.abs(fr)
    e_re = CF * (n_fft + 2) * U * (afr @ np.abs(cm).T)
    e_im = CF * (n_fft + 2) * U * (afr @ np.abs(sm).T)
    p = re * re + im * im
    e_p = 2 * np.abs(re) * e_re + 2 * np.abs(im) * e_im + e_re ** 2 + e_im ** 2 + CF * U * p
    if power == 2:
        spec, e_spec = p, e_p
    else:
        spec = np.sqrt(p)
        e_spec = np.minimum(e_p / np.maximum(spec, 1e-300), np.sqrt(e_p)) + CF * U * spec
    fbd = _f64(fb)
    mel = spec @ fbd.T
    e_mel = e_spec @ fbd.T + CF * (n_fft // 2 + 2) * U * mel
    fl = float(np.float32(floor_v))
    y = np.log(np.maximum(mel, fl))
    e_y = e_mel / np.maximum(mel - e_mel, fl) + CF * (2.0 ** -23 + 2 * U * np.abs(y))
    if div is not None:
        d = _f64(div)[None, :]
        y = y / d
        e_y = e_y / np.abs(d) + 2 * CF * U * np.abs(y)
    return y, e_y


def case_stft_mel(L, dev, T, cfg, n, signal, ldo=128):
    """ttb_audio_stft_mel on one signal: fp32 channel-major and bf16 token-major outputs between NaN canaries. Returns the
    error-to-bound ratios of the fp32 and of the bf16 output (the latter is dominated by the bf16 rounding itself)."""
    c = STFT_CONFIGS[cfg]
    n_mels, fb = c["n_mels"], T.fb[cfg]
    div = T.mel_norms if c["div"] else None
    x = stft_signal(signal, n)
    frames = 1 + n // T.hop
    of = torch.full((n_mels * frames + 61,), NAN, device=dev)
    ob = torch.full(((frames + 2) * ldo,), NAN, dtype=torch.bfloat16, device=dev)
    L.audio_stft_mel(x.to(dev), n, T.n_fft, T.hop, T.window, T.twiddle, fb, n_mels, c["power"], c["clip"], FLOOR, div,
                     out_bf16=ob, ldo=ldo, out_f32=of)
    want, bound = stft_mel64(x, T.n_fft, T.hop, T.window, T.twiddle, fb, c["power"], c["clip"], FLOOR, div)
    assert want.shape == (frames, n_mels)
    of, ob = of.cpu(), ob.cpu()
    name = "stft_mel %s n=%d %s" % (cfg, n, signal)
    untouched(name + " f32 tail", of[n_mels * frames:])
    untouched(name + " bf16 rows past the last frame", ob[frames * ldo:])
    got = of[:n_mels * frames].view(n_mels, frames).t()
    r32 = within(name + " f32", got, want, bound)
    gb = ob[:frames * ldo].view(frames, ldo)
    assert (gb[:, n_mels:].float() == 0).all(), name + ": bf16 columns n_mels..ldo-1 are not zero"
    rbf = within(name + " bf16", gb[:, :n_mels], want, bound + BF16_REL * (np.abs(want) + bound))
    if signal == "zeros":
        # digital silence: log(floor) [/ div] in every element, the same value in every frame
        assert torch.equal(got, got[:1].expand_as(got)), name + ": silence is not one value per channel"
    return r32, rbf


# ------------------------------------------------------------------ resampling
def resample_out_len(n, down, up):
    return -(-up * n // down)                                  # ceil(up * n / down)


def resample64(x, kern, down, up, width, m):
    """torchaudio.functional.resample's definition in float64 on the fp32 bank: pad by (width, width + down), correlate
    every phase j with kern[j] at stride down, interleave the phases (out[i * up + j]), keep the first m.
    Each output is a sum of klen products rounded once: bound c (klen + 1) u sum|terms|."""
    x, k = _f64(x), _f64(kern)
    klen = k.shape[1]
    xp = np.pad(x, (width, width + down))
    win = np.lib.stride_tricks.sliding_window_view(xp, klen)[::down]
    out = (win @ k.T).reshape(-1)
    s = (np.abs(win) @ np.abs(k).T).reshape(-1)
    assert m <= out.shape[0], (m, out.shape)
    return out[:m], CF * (klen + 1) * U * s[:m]


def resample_signal(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, generator=g) * 2 - 1
    x[-1] = 0.9                                                # a loud last sample: the tail past the input must see it
    return x


def case_resample(L, dev, T, ratio, n, m=None):
    """ttb_audio_resample: the m outputs wanted (default ceil(up n / down)) and nothing past them."""
    kern, down, up, width = T.resample[ratio]
    m = resample_out_len(n, down, up) if m is None else m
    x = resample_signal(n)
    out = torch.full((m + 67,), NAN, device=dev)
    L.audio_resample(x.to(dev), n, kern, down, up, kern.shape[1], width, out, m)
    want, bound = resample64(x, kern, down, up, width, m)
    out = out.cpu()
    name = "resample %d->%d n=%d m=%d" % (ratio[0], ratio[1], n, m)
    untouched(name + " past m", out[m:])
    return within(name, out[:m], want, bound)


# ------------------------------------------------------------------ means, EqualLinear
def case_mean_rows(L, dev, R, C, ld, accumulate, seed=0):
    """out[c] = (accumulate ? out[c] : 0) + scale * sum_r x[r * ld + c]. R + 1 roundings:
    bound c (R + 2) u (|scale| sum_r |x| + |out_before|)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(R * ld, generator=g) * 2 + 0.5
    scale = 1.0 / R if R > 1 else 0.37
    out = torch.full((C + 37,), NAN)
    prev = torch.zeros(C)
    if accumulate:
        prev = torch.randn(C, generator=g) * 3
        out[:C] = prev
    out = out.to(dev)
    L.mean_rows(x.to(dev), R, C, ld, scale, out, accumulate=accumulate)
    xs = _f64(x).reshape(R, ld)[:, :C]
    sc = float(np.float32(scale))
    pv = _f64(prev) if accumulate else 0.0
    want = pv + sc * xs.sum(0)
    bound = CF * (R + 2) * U * (abs(sc) * np.abs(xs).sum(0) + np.abs(pv))
    out = out.cpu()
    name = "mean_rows R=%d C=%d ld=%d acc=%d" % (R, C, ld, accumulate)
    untouched(name + " past C", out[C:])
    return within(name, out[:C], want, bound)


EQUAL_LINEAR_SETTINGS = {
    "equal_linear": lambda K: dict(wscale=(1 / math.sqrt(K)) * 0.1, bscale=0.1, slope=0.2, gain=2 ** 0.5),  # lr_mul 0.1
    "linear": lambda K: dict(wscale=1.0, bscale=1.0, slope=1.0, gain=1.0),                                   # nn.Linear
}


def case_equal_linear(L, dev, K, N, bias, settings, seed=0):
    """out = leaky_relu(x @ (W wscale)^T + b bscale, slope) gain. z is a sum of K products of x and the rounded W wscale
    plus the rounded b bscale: E_z = c (K + 2) u (sum|x W wscale| + |b bscale|); leaky_relu is Lipschitz with
    max(1, |slope|) and the gain product rounds once: bound |gain| max(1, |slope|) E_z + c u |out|."""
    g = torch.Generator().manual_seed(seed)
    s = EQUAL_LINEAR_SETTINGS[settings](K)
    x = torch.randn(K, generator=g)
    W = torch.randn(N, K, generator=g)
    b = torch.randn(N, generator=g) if bias else None
    out = torch.full((N + 29,), NAN, device=dev)
    L.equal_linear(x.to(dev), K, W.to(dev), None if b is None else b.to(dev), N, out, **s)
    f = {k: float(np.float32(v)) for k, v in s.items()}
    terms = _f64(x)[None, :] * _f64(W) * f["wscale"]
    bb = _f64(b) * f["bscale"] if bias else np.zeros(N)
    z = terms.sum(1) + bb
    want = np.where(z > 0, z, z * f["slope"]) * f["gain"]
    e_z = CF * (K + 2) * U * (np.abs(terms).sum(1) + np.abs(bb))
    bound = abs(f["gain"]) * max(1.0, abs(f["slope"])) * e_z + CF * U * np.abs(want)
    out = out.cpu()
    name = "equal_linear %s K=%d N=%d bias=%d" % (settings, K, N, bias)
    untouched(name + " past N", out[N:])
    return within(name, out[:N], want, bound)


# ------------------------------------------------------------------ CLVP pooling and projection
def clvp_pool64(x, g, b, eps=1e-5):
    """mean over T of LayerNorm(x[s, t]) g + b, x [nseq, T, D], and its bound. Per row:
    - mean: E_mu = c (D + 1) u sum|x| / D;
    - var = sum d^2 / D (d = x - mu): E_var = 2 E_mu sum|d| / D + c (D + 2) u var;
    - rstd = (var + eps)^-1/2: relative error E_var / (2 (var + eps)) + c u (approximate rsqrt);
    - z = d rstd: E_z = (E_mu + u|d|) rstd + |z| rel(rstd); y = z g + b: |g| E_z + c u (|z g| + |b|);
    - out = sum_t y / T over 8 warps' partial sums: E = sum_t E_y / T + c (T + 9) u sum_t |y| / T."""
    x, g, b = _f64(x), _f64(g), _f64(b)
    D = x.shape[-1]
    mu = x.mean(-1, keepdims=True)
    d = x - mu
    var = (d * d).mean(-1, keepdims=True)
    e_mu = CF * (D + 1) * U * np.abs(x).sum(-1, keepdims=True) / D
    e_var = 2 * e_mu * np.abs(d).sum(-1, keepdims=True) / D + CF * (D + 2) * U * var
    rstd = 1.0 / np.sqrt(var + eps)
    rel = e_var / (2 * (var + eps)) + CF * U
    z = d * rstd
    y = z * g + b
    e_z = (e_mu + U * np.abs(d)) * rstd + np.abs(z) * rel
    e_y = np.abs(g) * e_z + CF * U * (np.abs(z * g) + np.abs(b))
    T = x.shape[1]
    return y.mean(1), e_y.mean(1) + CF * (T + 9) * U * np.abs(y).mean(1)


def case_clvp_pool(L, dev, nseq, T, D, seed=0):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(nseq, T, D, generator=gen) * 2 + torch.randn(nseq, T, 1, generator=gen)
    g, b = 1 + torch.randn(D, generator=gen) * 0.2, torch.randn(D, generator=gen) * 0.2
    out = torch.full((nseq * D + 41,), NAN, device=dev)
    L.clvp_pool(x.reshape(-1).to(dev), nseq, T, D, g.to(dev), b.to(dev), out)
    want, bound = clvp_pool64(x, g, b)
    out = out.cpu()
    name = "clvp_pool nseq=%d T=%d D=%d" % (nseq, T, D)
    untouched(name + " past the last sequence", out[nseq * D:])
    return within(name, out[:nseq * D].view(nseq, D), want, bound)


def clvp_project64(pooled, W, text, temp):
    """latent = y / max(||y||, 1e-12) with y = pooled @ W^T, and score = <latent, text> temp.
    - y: D products per element: E_y = c (D + 1) u sum|W p|;
    - ||y||: by the triangle inequality the error of the exact norm is at most ||E_y||, plus c (D + 2) u ||y|| for the fp32
      sum of squares and the sqrt;
    - v = y / n: E_v = (E_y + |v| E_n) / (n - E_n) + c u |v|;
    - score: sum of D products and the temperature product: temp (sum E_v |t| + c (D + 2) u sum|v t|)."""
    p, W = _f64(pooled), _f64(W)
    y = p @ W.T
    e_y = CF * (W.shape[1] + 1) * U * (np.abs(p) @ np.abs(W).T)
    nrm = np.linalg.norm(y, axis=1, keepdims=True)
    e_n = np.linalg.norm(e_y, axis=1, keepdims=True) + CF * (W.shape[1] + 2) * U * nrm
    nd = np.maximum(nrm, 1e-12)
    v = y / nd
    e_v = (e_y + np.abs(v) * e_n) / np.maximum(nd - e_n, 1e-12) + CF * U * np.abs(v)
    if text is None:
        return v, e_v, None, None
    t = _f64(text)
    tf = float(np.float32(temp))
    s = (v @ t) * tf
    e_s = tf * (e_v @ np.abs(t) + CF * (W.shape[1] + 2) * U * (np.abs(v) @ np.abs(t)))
    return v, e_v, s, e_s


def case_clvp_project(L, dev, n, D, with_text, seed=0):
    """ttb_clvp_project with an all-zero pooled row (row 1), which F.normalize maps to a zero latent."""
    gen = torch.Generator().manual_seed(seed)
    pooled = torch.randn(n, D, generator=gen)
    pooled[1] = 0.0
    W = torch.randn(D, D, generator=gen) / math.sqrt(D)
    text = torch.nn.functional.normalize(torch.randn(D, generator=gen), dim=0) if with_text else None
    temp = math.exp(2.3)
    lat = torch.full((n * D + 19,), NAN, device=dev)
    sc = torch.full((n + 5,), NAN, device=dev)
    L.clvp_project(pooled.to(dev), n, D, W.to(dev), lat, None if text is None else text.to(dev), temp,
                   sc if with_text else None)
    v, e_v, s, e_s = clvp_project64(pooled, W, text, temp)
    lat, sc = lat.cpu(), sc.cpu()
    name = "clvp_project n=%d D=%d text=%d" % (n, D, with_text)
    untouched(name + " latents past n", lat[n * D:])
    lv = lat[:n * D].view(n, D)
    r = within(name + " latents", lv, v, e_v)
    assert (lv[1] == 0).all(), name + ": the all-zero row did not give a zero latent"
    if with_text:
        untouched(name + " scores past n", sc[n:])
        r = max(r, within(name + " scores", sc[:n], s, e_s))
        assert sc[1].item() == 0.0
    else:
        untouched(name + " scores (not requested)", sc)
    return r


# ------------------------------------------------------------------ exact kernels (bit for bit)
def case_exact_kernels(L, dev, seed=0):
    """ttb_embed, ttb_cast_pad_bf16, ttb_broadcast_rows, ttb_voc_to_tokens_bf16, ttb_transpose_f32 and ttb_counter_add
    against torch on the same fp32 values (one fp32 add, or torch's round-to-nearest bf16 cast)."""
    gen = torch.Generator().manual_seed(seed)
    bf = torch.bfloat16

    def rn(*s):
        return torch.randn(*s, generator=gen) * 3

    # embed: rows of a table (+ a positional table), ragged D
    n, D = 13, 197
    table, pos_table = rn(50, D), rn(40, D)
    ids = torch.randint(0, 50, (n,), generator=gen, dtype=torch.int32)
    pos = torch.randint(0, 40, (n,), generator=gen, dtype=torch.int32)
    for with_pos in (True, False):
        out = torch.full((n * D + 23,), NAN, device=dev)
        L.embed(ids.to(dev), pos.to(dev) if with_pos else None, n, D, table.to(dev), pos_table.to(dev), out)
        want = table[ids.long()] + (pos_table[pos.long()] if with_pos else 0.0)
        out = out.cpu()
        assert torch.equal(out[:n * D].view(n, D), want), "embed pos=%d" % with_pos
        untouched("embed past n", out[n * D:])
    # cast_pad_bf16: rows of stride ld_in -> bf16 rows of stride ldo, columns Cc..ncols-1 zero, ncols..ldo-1 untouched
    R, Cc, ld_in, ncols, ldo = 19, 37, 45, 50, 56
    src = rn(R * ld_in)
    out = torch.full((R * ldo + 9,), NAN, dtype=bf, device=dev)
    L.cast_pad_bf16(src.to(dev), R, Cc, ld_in, out, ldo, ncols)
    out = out.cpu()
    o = out[:R * ldo].view(R, ldo)
    assert torch.equal(o[:, :Cc], src.view(R, ld_in)[:, :Cc].to(bf)), "cast_pad_bf16 values"
    assert (o[:, Cc:ncols].float() == 0).all(), "cast_pad_bf16 zero fill"
    untouched("cast_pad_bf16 columns past ncols", o[:, ncols:])
    untouched("cast_pad_bf16 past R", out[R * ldo:])
    # broadcast_rows: fp32 and bf16 copies of one row, columns Cc..ldo-1 untouched; either output alone
    row = rn(Cc)
    for f32, b16 in ((True, True), (True, False), (False, True)):
        of = torch.full((R * ldo + 9,), NAN, device=dev)
        ob = torch.full((R * ldo + 9,), NAN, dtype=bf, device=dev)
        L.broadcast_rows(row.to(dev), R, Cc, of if f32 else None, ob if b16 else None, ldo)
        of, ob = of.cpu(), ob.cpu()
        for on, buf, want in ((f32, of, row), (b16, ob, row.to(bf))):
            if not on:
                untouched("broadcast_rows output not requested", buf)
                continue
            v = buf[:R * ldo].view(R, ldo)
            assert torch.equal(v[:, :Cc], want.expand(R, Cc)), "broadcast_rows values %s" % buf.dtype
            untouched("broadcast_rows columns past Cc", v[:, Cc:])
            untouched("broadcast_rows past R", buf[R * ldo:])
    # voc_to_tokens_bf16: channel-major [C, L] -> token-major; C and L not multiples of 32
    C2, L2 = 37, 45
    x = rn(C2, L2) * torch.exp(rn(C2, L2))        # magnitudes over many binades
    xt = x.t()
    hi = xt.to(bf)
    lo = (xt - hi.float()).to(bf)
    ldo2 = 40
    out = torch.full((L2 * ldo2 + 7,), NAN, dtype=bf, device=dev)
    L.voc_to_tokens_bf16(x.reshape(-1).to(dev), C2, L2, out, ldo2, split=False)
    out = out.cpu()
    o = out[:L2 * ldo2].view(L2, ldo2)
    assert torch.equal(o[:, :C2], hi), "voc_to_tokens hi"
    assert (o[:, C2:].float() == 0).all(), "voc_to_tokens zero columns"
    untouched("voc_to_tokens past L", out[L2 * ldo2:])
    ldo3 = 3 * C2 + 13
    out = torch.full((L2 * ldo3 + 7,), NAN, dtype=bf, device=dev)
    L.voc_to_tokens_bf16(x.reshape(-1).to(dev), C2, L2, out, ldo3, split=True)
    out = out.cpu()
    o = out[:L2 * ldo3].view(L2, ldo3)
    assert torch.equal(o[:, :C2], hi), "voc_to_tokens split hi"
    assert torch.equal(o[:, C2:2 * C2], lo), "voc_to_tokens split lo = bf16(v - hi)"
    assert torch.equal(o[:, 2 * C2:3 * C2], hi), "voc_to_tokens split third block"
    untouched("voc_to_tokens split columns past 3C", o[:, 3 * C2:])
    untouched("voc_to_tokens split past L", out[L2 * ldo3:])
    v64 = _f64(xt)
    assert (np.abs(_f64(o[:, :C2]) + _f64(o[:, C2:2 * C2]) - v64) <= 2.0 ** -16 * np.abs(v64)).all(), \
        "voc_to_tokens split: hi + lo is not v to 2^-16"
    # transpose_f32 at ragged sizes
    for R3, C3 in ((1, 1), (1, 70), (33, 65), (100, 37), (31, 33)):
        a = rn(R3, C3)
        out = torch.full((R3 * C3 + 11,), NAN, device=dev)
        L.transpose_f32(a.reshape(-1).to(dev), R3, C3, out)
        out = out.cpu()
        assert torch.equal(out[:R3 * C3].view(C3, R3), a.t()), "transpose %dx%d" % (R3, C3)
        untouched("transpose past R*C", out[R3 * C3:])
    # counter_add: one int, its neighbours unchanged
    ctr = torch.tensor([-7, 5, 11], dtype=torch.int32, device=dev)
    L.counter_add(ctr[1:], 3)
    L.counter_add(ctr[1:], -1)
    assert ctr.cpu().tolist() == [-7, 7, 11]

