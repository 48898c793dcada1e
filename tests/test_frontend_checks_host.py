"""CPU: the float64 references and bounds of frontend_checks.py accept an fp32 implementation of each kernel (the torch
emulation of tests/lib_emu.py) and reject subtly wrong versions of the same computation, run through the same cases
the GPU tests run."""
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import frontend_checks as fc
import lib_emu


@pytest.fixture(scope="module")
def tables():
    return fc.Tables("cpu")


def _stft_fp32(x, n, n_fft, hop, window, twiddle, fb, n_mels, power, clip, floor_v, div, out_bf16=None, ldo=0,
               out_f32=None, pad_shift=0, drop_last=False, ignore_clip=False):
    """lib_emu.audio_stft_mel with one mistake switched on: reflect padding that repeats the edge sample (pad_shift=1),
    the last frame not computed, or `clip` ignored."""
    v = x[:n].clamp(-1, 1) if clip and not ignore_clip else x[:n]
    p, s = n_fft // 2, pad_shift
    xp = torch.cat([v[1 - s:p + 1 - s].flip(0), v, v[n - 1 - p + s:n - 1 + s].flip(0)])
    fr = xp.unfold(0, n_fft, hop) * window
    if drop_last:
        fr = fr[:-1]
    idx = (torch.arange(n_fft // 2 + 1)[:, None] * torch.arange(n_fft)[None, :]) % n_fft
    re, im = fr @ twiddle[:, 0][idx].t(), -(fr @ twiddle[:, 1][idx].t())
    p2 = re * re + im * im
    y = torch.log(((p2 if power == 2 else p2.sqrt()) @ fb.t()).clamp(min=floor_v))
    if div is not None:
        y = y / div
    frames = y.shape[0]
    full = 1 + n // hop
    if out_f32 is not None:
        lib_emu._v(out_f32, (n_mels, frames), (full, 1)).copy_(y.t())
    if out_bf16 is not None:
        o = lib_emu._v(out_bf16, (frames, ldo), (ldo, 1))
        o.zero_()
        o[:, :n_mels] = y.to(torch.bfloat16)


def _mutant(**fns):
    m = types.SimpleNamespace(**{k: getattr(lib_emu, k) for k in dir(lib_emu) if not k.startswith("_")})
    for k, v in fns.items():
        setattr(m, k, v)
    return m


def _resample_tail_truncated(x, n, kernels, down, up, klen, width, out, m):
    """Outputs whose window reaches past the last input sample are left at zero."""
    lib_emu.audio_resample(x, n, kernels, down, up, klen, width, out, m)
    i = torch.arange(m) // up
    out[:m][i * down - width + klen > n] = 0.0


def _mean_rows_no_accumulate(x, R, Cc, ld, scale, out, accumulate=False):
    lib_emu.mean_rows(x, R, Cc, ld, scale, out, accumulate=False)


def _to_tokens_lo_from_v(x, Cc, L, out, ldo, split=False):
    lib_emu.voc_to_tokens_bf16(x, Cc, L, out, ldo, split)
    if split:
        o = lib_emu._v(out, (L, ldo), (ldo, 1))
        o[:, Cc:2 * Cc] = lib_emu._v(x, (Cc, L), (L, 1)).t().to(torch.bfloat16)


def _cast_pad_no_zero_fill(inp, R, Cc, ld_in, out, ldo, ncols_out=None):
    lib_emu._v(out, (R, Cc), (ldo, 1)).copy_(lib_emu._v(inp, (R, Cc), (ld_in, 1)).to(torch.bfloat16))


def _normalize_without_eps_guard(pooled, n, D, W, latents, text_latent, temp_exp, scores):
    y = lib_emu._v(pooled, (n, D), (D, 1)) @ W.t()
    y = y / y.norm(dim=-1, keepdim=True)
    lib_emu._v(latents, (n, D), (D, 1)).copy_(y)
    if text_latent is not None:
        scores[:n] = (y @ text_latent.reshape(-1)) * temp_exp


def _stft_case(cfg, n, sig):
    return lambda L, T: fc.case_stft_mel(L, "cpu", T, cfg, n, sig)


# (mutant, the case that must reject it)
MUTANTS = {
    "reflect padding off by one, first frame": (_mutant(audio_stft_mel=lambda *a, **k: _stft_fp32(*a, pad_shift=1, **k)),
                                                _stft_case("ar", 513, "impulse1")),
    "reflect padding off by one, last frame": (_mutant(audio_stft_mel=lambda *a, **k: _stft_fp32(*a, pad_shift=1, **k)),
                                               _stft_case("diffusion", 10239, "impulse_n2")),
    "last frame dropped": (_mutant(audio_stft_mel=lambda *a, **k: _stft_fp32(*a, drop_last=True, **k)),
                           _stft_case("diffusion", 10240, "noise")),
    "clip ignored": (_mutant(audio_stft_mel=lambda *a, **k: _stft_fp32(*a, ignore_clip=True, **k)),
                     _stft_case("diffusion", 1024, "loud")),
    "resampler tail truncated": (_mutant(audio_resample=_resample_tail_truncated),
                                 lambda L, T: fc.case_resample(L, "cpu", T, (24000, 16000), 5000)),
    "resampler tail truncated, short input": (_mutant(audio_resample=_resample_tail_truncated),
                                              lambda L, T: fc.case_resample(L, "cpu", T, (22050, 24000), 7)),
    "accumulate ignored": (_mutant(mean_rows=_mean_rows_no_accumulate),
                           lambda L, T: fc.case_mean_rows(L, "cpu", 37, 300, 333, True)),
    "lo computed from v instead of v - hi": (_mutant(voc_to_tokens_bf16=_to_tokens_lo_from_v),
                                             lambda L, T: fc.case_exact_kernels(L, "cpu")),
    "cast_pad_bf16 without the zero fill": (_mutant(cast_pad_bf16=_cast_pad_no_zero_fill),
                                            lambda L, T: fc.case_exact_kernels(L, "cpu")),
    "normalize without the 1e-12 floor": (_mutant(clvp_project=_normalize_without_eps_guard),
                                          lambda L, T: fc.case_clvp_project(L, "cpu", 6, 512, True)),
}


def test_emulation_meets_every_bound(tables):
    """An fp32 implementation of each kernel passes: the bounds are not tighter than fp32 arithmetic."""
    for cfg in sorted(fc.STFT_CONFIGS):
        for n in (513, 10239, 10240):
            for sig in fc.STFT_SIGNALS:
                fc.case_stft_mel(lib_emu, "cpu", tables, cfg, n, sig)
    for ratio in fc.RESAMPLE_RATIOS:
        for n in (1, 7, 5000):
            fc.case_resample(lib_emu, "cpu", tables, ratio, n)
        fc.case_resample(lib_emu, "cpu", tables, ratio, 5000, 3000)
    for acc in (False, True):
        fc.case_mean_rows(lib_emu, "cpu", 37, 300, 333, acc)
        fc.case_mean_rows(lib_emu, "cpu", 1, 300, 301, acc)
    for s in fc.EQUAL_LINEAR_SETTINGS:
        fc.case_equal_linear(lib_emu, "cpu", 300, 77, True, s)
        fc.case_equal_linear(lib_emu, "cpu", 31, 5, False, s)
    fc.case_clvp_pool(lib_emu, "cpu", 3, 13, 768)
    fc.case_clvp_project(lib_emu, "cpu", 6, 512, True)
    fc.case_clvp_project(lib_emu, "cpu", 6, 512, False)
    fc.case_exact_kernels(lib_emu, "cpu")


@pytest.mark.parametrize("name", sorted(MUTANTS))
def test_mutant_rejected(tables, name):
    mutant, case = MUTANTS[name]
    with pytest.raises(AssertionError):
        case(mutant, tables)


def test_stft_reference_is_torch_stft():
    """The float64 STFT restatement agrees with torch.stft (center, reflect) on the same fp32 window, to the rounding of
    the fp32 twiddles."""
    T = fc.Tables("cpu")
    x = fc.stft_signal("noise", 5000)
    want, _ = fc.stft_mel64(x, 1024, 256, T.window, T.twiddle, torch.eye(513), 2, False, 1e-30, None)
    s = torch.stft(x.double(), 1024, 256, window=T.window.double(), center=True, pad_mode="reflect", return_complex=True)
    p = s.abs().pow(2).t().numpy()
    np.testing.assert_allclose(np.exp(want), p, rtol=0, atol=1e-6 * p.max())


def test_resample_reference_is_conv1d():
    """The float64 resampling restatement agrees with torchaudio's padded strided conv1d on the same bank."""
    T = fc.Tables("cpu")
    for (orig, new), (k, down, up, width) in T.resample.items():
        x = fc.resample_signal(777)
        m = fc.resample_out_len(777, down, up)
        want, _ = fc.resample64(x, k, down, up, width, m)
        y = F.conv1d(F.pad(x.double().reshape(1, 1, -1), (width, width + down)), k.double()[:, None, :], stride=down)
        np.testing.assert_allclose(want, y[0].t().reshape(-1)[:m].numpy(), rtol=0, atol=1e-12)
