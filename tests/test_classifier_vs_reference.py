"""CPU, reference: oracle/classifier.py against the unmodified AudioMiniEncoderWithClassifierHead that
`classify_audio_clip` builds (tortoise/api.py:133-145), loaded strictly with synth_classifier weights."""
import pytest
import torch

from oracle import classifier as oc
from tortoise_tts_b200.synth import synth_classifier
from test_classifier_host import make_clip

pytestmark = pytest.mark.reference


@pytest.fixture(scope="module")
def ref_model():
    from oracle.ref_shims import load_reference
    load_reference()
    from tortoise.models.classifier import AudioMiniEncoderWithClassifierHead
    m = AudioMiniEncoderWithClassifierHead(2, spec_dim=1, embedding_dim=512, depth=5, downsample_factor=4,
                                           resnet_blocks=2, attn_blocks=4, num_attn_heads=4, base_channels=32,
                                           dropout=0, kernel_size=5, distribute_zero_label=False)
    sd = synth_classifier(0)
    m.load_state_dict(sd, strict=True)
    return m.eval(), sd


@pytest.mark.parametrize("n", [220000, 99001, 2049])
def test_oracle_matches_reference(ref_model, n):
    m, sd = ref_model
    clip = make_clip(n)
    with torch.no_grad():
        want = m(clip.unsqueeze(0))                            # as classify_audio_clip: [1, n] -> [1, 1, n]
        got = oc.logits(sd, clip)
    assert got.shape == want.shape == (1, 2)
    assert (got - want).abs().max().item() < 1e-5
    assert abs(oc.classify(sd, clip).item() - torch.softmax(want, -1)[0][0].item()) < 1e-5
