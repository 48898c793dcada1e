"""GPU: the conditioning front-end (ttb_audio_stft_mel, ttb_audio_resample) and the small helper kernels behind the
C-ABI against float64 restatements of their definitions, per element, between NaN canaries.

The references, the bounds and their reasoning are in frontend_checks.py; each case there asserts that every documented
output element is written and within its bound, and that nothing past the documented region changes. The largest error
relative to its bound is reported for every case. test_frontend_checks_host.py shows that each bound rejects a subtly
wrong version of the same computation.
"""
import pytest
import torch

import frontend_checks as fc
from gpu_util import report

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    from tortoise_tts_b200 import lib
    return lib


@pytest.fixture(scope="module")
def tables():
    return fc.Tables("cuda")


def _stft_lengths(cfg):
    hop = 256
    return (1024 // 2 + 1, 1024, 40 * hop, 40 * hop - 1, fc.STFT_CONFIGS[cfg]["prod_n"])


@pytest.mark.parametrize("cfg", sorted(fc.STFT_CONFIGS))
def test_stft_mel(lib, tables, cfg):
    """Both production configurations (AR: 80 mels, power 2, / mel_norms; diffusion: 100 mels, power 1, clip) at the
    shortest accepted length, 1024, a multiple of hop, a multiple of hop minus 1 and the production length, on silence,
    impulses at both ends, a burst, a DC offset, samples up to +-3 and full-scale noise."""
    w32 = wbf = 0.0
    for n in _stft_lengths(cfg):
        for sig in fc.STFT_SIGNALS:
            r32, rbf = fc.case_stft_mel(lib, "cuda", tables, cfg, n, sig)
            w32, wbf = max(w32, r32), max(wbf, rbf)
    report("stft_mel %s fp32 output vs float64 (error / bound)" % cfg, w32)
    report("stft_mel %s bf16 output vs float64 (error / bound)" % cfg, wbf)


def test_stft_mel_errors(lib, tables):
    """Shapes the kernel does not take return an error instead of launching."""
    x = torch.zeros(4096, device="cuda")
    out = torch.full((17 * 128,), float("nan"), dtype=torch.bfloat16, device="cuda")
    fb = tables.fb["ar"]
    args = dict(out_bf16=out, ldo=128)
    with pytest.raises(lib.TtbError):
        lib.audio_stft_mel(x, 512, 1024, 256, tables.window, tables.twiddle, fb, 80, 2, False, 1e-5, None, **args)
    with pytest.raises(lib.TtbError):
        lib.audio_stft_mel(x, 4096, 1000, 256, tables.window, tables.twiddle, fb, 80, 2, False, 1e-5, None, **args)
    for power in (0, 3):
        with pytest.raises(lib.TtbError):
            lib.audio_stft_mel(x, 4096, 1024, 256, tables.window, tables.twiddle, fb, 80, power, False, 1e-5, None, **args)
    torch.cuda.synchronize()
    assert torch.isnan(out.float()).all()


@pytest.mark.parametrize("ratio", fc.RESAMPLE_RATIOS, ids=lambda r: "%d-%d" % r)
def test_resample(lib, tables, ratio):
    """22050 -> 24000 (diffusion conditioning) and 24000 -> 16000 (wav2vec): one sample, fewer samples than the kernel
    is long, a clip whose every output is wanted, and the truncated case (the 102400 cap of diffusion_mel)."""
    kern, down, up, width = tables.resample[ratio]
    klen = kern.shape[1]
    worst = 0.0
    for n in (1, 7, klen - 3, klen + 1, 5000, 100003):
        worst = max(worst, fc.case_resample(lib, "cuda", tables, ratio, n))
    n = 100000
    m_full = fc.resample_out_len(n, down, up)
    m = 102400 if m_full > 102400 else m_full - 777
    worst = max(worst, fc.case_resample(lib, "cuda", tables, ratio, n, m))
    report("resample %d->%d vs float64 (error / bound)" % ratio, worst)


def test_mean_rows(lib):
    worst = 0.0
    for R, C, ld in ((1, 1024, 1024), (1, 300, 301), (37, 300, 333), (401, 2048, 2048), (5, 257, 1024)):
        for acc in (False, True):
            worst = max(worst, fc.case_mean_rows(lib, "cuda", R, C, ld, acc))
    report("mean_rows vs float64 (error / bound)", worst)


def test_equal_linear(lib):
    """The random-voice converter's EqualLinear settings and plain nn.Linear, with and without a bias, at K not a
    multiple of 32 and N not a multiple of 8."""
    worst = 0.0
    for settings in sorted(fc.EQUAL_LINEAR_SETTINGS):
        for K, N in ((1024, 1024), (300, 77), (31, 5)):
            for bias in (True, False):
                worst = max(worst, fc.case_equal_linear(lib, "cuda", K, N, bias, settings))
    report("equal_linear vs float64 (error / bound)", worst)


@pytest.mark.parametrize("D", [512, 768, 1024])
def test_clvp_pool(lib, D):
    worst = 0.0
    for nseq, T in ((1, 1), (3, 13), (2, 8), (4, 250)):
        worst = max(worst, fc.case_clvp_pool(lib, "cuda", nseq, T, D))
    report("clvp_pool D=%d vs float64 (error / bound)" % D, worst)


@pytest.mark.parametrize("D", [512, 768, 1024])
def test_clvp_project(lib, D):
    worst = 0.0
    for with_text in (True, False):
        worst = max(worst, fc.case_clvp_project(lib, "cuda", 6, D, with_text))
    report("clvp_project D=%d vs float64 (error / bound)" % D, worst)


def test_exact_kernels(lib):
    fc.case_exact_kernels(lib, "cuda")
