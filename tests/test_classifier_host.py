"""CPU: the classifier engine's orchestration (weight packing, conv taps, the K-padded level 0, the quad-view
Downsample, attention layout) under the torch emulation of libttb.so (tests/lib_emu.py), against the fp32 oracle; and
the checks on inputs that reach the engine from outside.

The emulation rounds GEMM operands and the attention's q / k / v to bf16 as the kernels do, so the difference it shows
against the fp32 oracle is the drift that bf16 operands cause. DRIFT_* below is that measured drift with a margin, and
tests/test_gpu_classifier.py uses the same bounds for the kernels."""
import pytest
import torch

from oracle import classifier as oc
from tortoise_tts_b200.synth import synth_classifier

LENGTHS = (220000, 99001, 2049)

# bf16 rounding makes the drift a noisy quantity: a relative change of 1e-6 in the input can move it several-fold. So it is
# measured over several clips and input perturbations (test_engine_matches_oracle_under_emulation: 2 weight seeds x
# 3 lengths x 4 clips x 2 perturbations). Measured maxima: logit |diff| 3.1e-2 (n = 2049, where only T = 3
# positions reach the head), |diff| / max |logit| 4.8e-2, probability |diff| 6.0e-3; a wider scan at n = 2049 and
# 99 001 (8 clips, perturbations of +-1e-6) gave at most 3.1e-2, 5.4e-2 and 6.0e-3. The bounds are about twice that.
DRIFT_LOGIT = 6e-2
DRIFT_LOGIT_REL = 0.1
DRIFT_PROB = 1.2e-2


def make_clip(n, seed=0):
    """A 24 kHz test clip: a tone plus noise, amplitude well inside [-1, 1]."""
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(n) / 24000.0
    return (0.3 * torch.sin(2 * torch.pi * (150 + 50 * seed) * t) + 0.1 * torch.randn(n, generator=g)).reshape(1, n)



@pytest.fixture(scope="module")
def emu():
    import lib_emu
    saved = lib_emu.install()
    yield
    lib_emu.uninstall(saved)


@pytest.mark.parametrize("seed", [0, 1])
def test_engine_matches_oracle_under_emulation(emu, seed):
    from tortoise_tts_b200.classifier_engine import ClassifierEngine
    sd = synth_classifier(seed)
    eng = ClassifierEngine(sd, device="cpu")
    for n in LENGTHS:
        worst = [0.0, 0.0, 0.0]
        for clip_seed in range(4):
            for eps in (0.0, 1e-6):
                clip = make_clip(n, clip_seed) * (1 + eps)
                want = oc.logits(sd, clip)
                pw = torch.softmax(want, -1)
                assert 0.05 < pw[0, 0].item() < 0.95, (n, clip_seed, pw)      # the softmax is not saturated
                got, probs = eng.forward(clip)
                dl = (got - want).abs().max().item()
                d = (dl, dl / want.abs().max().item(), (probs - pw).abs().max().item())
                worst = [max(a, b) for a, b in zip(worst, d)]
                assert d[0] < DRIFT_LOGIT and d[1] < DRIFT_LOGIT_REL and d[2] < DRIFT_PROB, (n, clip_seed, eps, d)
        print("seed %d n %d: max logit diff %.2e (rel %.2e), max prob diff %.2e" % (seed, n, *worst))


def test_level_lengths_and_quad_view_padding():
    from tortoise_tts_b200.classifier_engine import level_lengths
    assert level_lengths(220000) == [220000, 55000, 13750, 3438, 860, 215]
    assert level_lengths(99001) == [99001, 24751, 6188, 1547, 387, 97]
    assert level_lengths(2049) == [2049, 513, 129, 33, 9, 3]
    for n in (220000, 99001, 2049, 5):
        L = n
        for Lq in level_lengths(n)[1:]:
            assert Lq == (L + 2 * 2 - 5) // 4 + 1                   # Conv1d(k5, stride 4, pad 2)
            L = Lq


def test_rejects_other_architectures():
    from tortoise_tts_b200.classifier_engine import check_state_dict
    sd = synth_classifier(0)
    check_state_dict(sd)
    bad = dict(sd)
    bad["enc.res.0.in_layers.2.weight"] = torch.zeros(32, 32, 3)
    with pytest.raises(ValueError, match="in_layers.2.weight has shape"):
        check_state_dict(bad)
    bad = dict(sd)
    del bad["head.bias"]
    with pytest.raises(ValueError, match="missing head.bias"):
        check_state_dict(bad)
    bad = dict(sd)
    bad["enc.res.15.op.weight"] = torch.zeros(1)
    with pytest.raises(ValueError, match="unexpected"):
        check_state_dict(bad)


@pytest.mark.parametrize("clip", [torch.zeros(5), torch.zeros(2, 5), torch.zeros(1, 1, 5), torch.zeros(1, 0),
                                  torch.zeros(1, 5, dtype=torch.int32), [[0.0] * 5]])
def test_facade_rejects_other_shapes(clip):
    from tortoise_tts_b200.api import classify_audio_clip
    with pytest.raises(ValueError, match=r"\[1, n\]"):
        classify_audio_clip(clip, models_dir="/nonexistent")


def test_api_fast_reexports():
    from tortoise_tts_b200 import api, api_fast
    assert api_fast.classify_audio_clip is api.classify_audio_clip
