"""GPU: GroupNorm with 2 channels per group against float64 torch, and the classifier engine and
`classify_audio_clip` against the fp32 oracle (oracle/classifier.py) within the bf16-operand drift that
tests/test_classifier_host.py measures."""
import pytest
import torch
import torch.nn.functional as F

from gpu_util import report
from oracle import classifier as oc
from test_classifier_host import DRIFT_LOGIT, DRIFT_LOGIT_REL, DRIFT_PROB, make_clip
from tortoise_tts_b200.synth import synth_classifier

pytestmark = pytest.mark.gpu


def _gn_inputs(B, S, C, seed):
    g = torch.Generator().manual_seed(seed)
    std = 0.5 + torch.rand(C, generator=g)
    off = (torch.rand(C, generator=g) * 2 - 1) * std             # per-channel offsets up to one standard deviation
    x = torch.randn(B, S, C, generator=g) * std + off
    gamma, beta = 1 + 0.1 * torch.randn(C, generator=g), 0.1 * torch.randn(C, generator=g)
    return x, gamma, beta


@pytest.mark.parametrize("S", [220000, 99001, 7])
@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("silu", [False, True])
def test_groupnorm_two_channels_per_group(S, B, silu):
    from tortoise_tts_b200 import lib
    C, G = 32, 16
    x, gamma, beta = _gn_inputs(B, S, C, S + B)
    want = F.group_norm(x.double().transpose(1, 2), G, gamma.double(), beta.double(), 1e-5).transpose(1, 2)
    if silu:
        want = F.silu(want)
    xc, gc, bc = x.cuda(), gamma.cuda(), beta.cuda()
    part = lib.groupnorm_scratch(B, G, "cuda")
    ob = torch.full((B, S, 64), 7.0, dtype=torch.bfloat16, device="cuda")
    of = torch.empty(B, S, C, device="cuda")
    lib.groupnorm(xc, B, S, C, G, gc, bc, part, silu=silu, out_bf16=ob, ldo=64, out_f32=of, ldof=C)
    ef = (of.double().cpu() - want).abs().max().item()
    eb = ((ob[..., :C].double().cpu() - want).abs() - want.abs() * 2 ** -8).max().item()
    report("groupnorm cpg 2 S=%d B=%d silu=%d fp32" % (S, B, silu), ef)
    report("groupnorm cpg 2 S=%d B=%d silu=%d bf16 (beyond half an ulp)" % (S, B, silu), eb)
    assert ef < 1e-4
    assert eb < 1e-4
    assert bool((ob[..., C:] == 7.0).all())                        # columns C..ldo-1 are not written
    # bf16 only, then fp32 only: the same values, and bit-identical to the first call
    ob2 = torch.zeros(B, S, 64, dtype=torch.bfloat16, device="cuda")
    lib.groupnorm(xc, B, S, C, G, gc, bc, part, silu=silu, out_bf16=ob2, ldo=64)
    of2 = torch.zeros(B, S, C, device="cuda")
    lib.groupnorm(xc, B, S, C, G, gc, bc, part, silu=silu, out_f32=of2, ldof=C)
    assert torch.equal(ob2[..., :C], ob[..., :C]) and torch.equal(of2, of)


def test_groupnorm_two_channels_per_group_rejects_what_it_lacks():
    from tortoise_tts_b200 import lib
    S, C, G = 64, 32, 16
    x, gamma, beta = (t.cuda() for t in _gn_inputs(1, S, C, 0))
    part = lib.groupnorm_scratch(1, G, "cuda")
    out = torch.empty(S, C, device="cuda")
    ss = torch.zeros(1, 2 * C, device="cuda")
    with pytest.raises(lib.TtbError, match="2 channels per group"):
        lib.groupnorm(x, 1, S, C, G, gamma, beta, part, scale_shift=ss, ss_bstride=2 * C, out_f32=out, ldof=C)
    x48 = torch.zeros(S, 48, device="cuda")
    g48 = torch.ones(48, device="cuda")
    with pytest.raises(lib.TtbError, match="2 channels per group"):
        lib.groupnorm(x48, 1, S, 48, 24, g48, g48, part, out_f32=torch.empty(S, 48, device="cuda"), ldof=48)


@pytest.fixture(scope="module")
def engines():
    from tortoise_tts_b200.classifier_engine import ClassifierEngine
    out = {}
    for seed in (0, 1):
        sd = synth_classifier(seed)
        out[seed] = (sd, ClassifierEngine(sd, device="cuda"))
    return out


@pytest.mark.parametrize("n", [220000, 99001, 2049, 480000])
@pytest.mark.parametrize("seed", [0, 1])
def test_engine_matches_oracle(engines, n, seed):
    sd, eng = engines[seed]
    clip = make_clip(n, seed)
    want = oc.logits(sd, clip)
    pw = torch.softmax(want, -1)
    logits, probs = eng.forward(clip.cuda())
    dl = (logits.cpu() - want).abs().max().item()
    rel = dl / want.abs().max().item()
    dp = (probs.cpu() - pw).abs().max().item()
    report("classifier logits n=%d seed=%d (bound %.0e)" % (n, seed, DRIFT_LOGIT), dl)
    report("classifier logits rel n=%d seed=%d (bound %.0e)" % (n, seed, DRIFT_LOGIT_REL), rel)
    report("classifier prob n=%d seed=%d (bound %.0e)" % (n, seed, DRIFT_PROB), dp)
    assert dl < DRIFT_LOGIT and rel < DRIFT_LOGIT_REL and dp < DRIFT_PROB


def test_engine_is_deterministic(engines):
    _, eng = engines[0]
    clip = make_clip(99001, 3).cuda()
    a = eng.forward(clip)
    b = eng.forward(clip)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_classify_audio_clip(engines, tmp_path):
    from tortoise_tts_b200 import api, api_fast
    sd, eng = engines[1]
    torch.save(sd, tmp_path / "classifier.pth")
    clip = make_clip(2049, 5)
    p = api.classify_audio_clip(clip, models_dir=str(tmp_path))
    assert p.dim() == 0 and p.dtype == torch.float32 and p.device.type == "cpu"
    assert torch.equal(p, eng.forward(clip.cuda())[1][0, 0].cpu())
    assert abs(p.item() - oc.classify(sd, clip).item()) < DRIFT_PROB
    cached = dict(api._CLASSIFIERS)
    p2 = api_fast.classify_audio_clip(clip.cuda(), models_dir=str(tmp_path))   # any device; the engine is reused
    assert torch.equal(p, p2) and api._CLASSIFIERS == cached
