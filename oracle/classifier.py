"""TEST INFRASTRUCTURE ONLY (CPU oracle) — restatement of the tortoise-detect classifier that
`tortoise/api.py:133-145` (`classify_audio_clip`) runs: AudioMiniEncoderWithClassifierHead(2, spec_dim=1,
embedding_dim=512, depth=5, downsample_factor=4, resnet_blocks=2, attn_blocks=4, num_attn_heads=4, base_channels=32,
kernel_size=5) in eval mode.

Plain torch-fp32 functional code over the reference `classifier.pth` state_dict (models/classifier.py):
  init: Conv1d(1, 32, k3, p1)                                                                      (classifier.py:92-94)
  5 levels, C = 32 * 2^l: 2 x ResBlock  x + conv5(SiLU(GN(conv5(SiLU(GN(x))))))  (identity skip)  (classifier.py:7-77)
                          Downsample    Conv1d(C, 2C, k5, stride 4, p2)                            (arch_util.py:153-178)
  final: GN(1024) -> SiLU -> Conv1d(1024, 512, k1)                                                 (classifier.py:103-107)
  4 x AttentionBlock(512, 4 heads, no relative positions) -> position 0 -> Linear(512, 2)         (classifier.py:108-141)
Pinned against the reference module by tests/test_classifier_vs_reference.py.
"""
import torch
import torch.nn.functional as F

from .diffusion import _gn, attention_block

DEPTH, RESNET_BLOCKS, ATTN_BLOCKS, HEADS = 5, 2, 4, 4


def logits(sd, clip):
    """clip: waveform [1, n] (or [n]) -> logits fp32 [1, 2] (AudioMiniEncoderWithClassifierHead.forward)."""
    h = F.conv1d(clip.reshape(1, 1, -1).float(), sd["enc.init.0.weight"], sd["enc.init.0.bias"], padding=1)
    i = 0
    for _ in range(DEPTH):
        for _ in range(RESNET_BLOCKS):
            p = f"enc.res.{i}."
            t = F.conv1d(F.silu(_gn(h, sd[p + "in_layers.0.weight"], sd[p + "in_layers.0.bias"])),
                         sd[p + "in_layers.2.weight"], sd[p + "in_layers.2.bias"], padding=2)
            t = F.conv1d(F.silu(_gn(t, sd[p + "out_layers.0.weight"], sd[p + "out_layers.0.bias"])),
                         sd[p + "out_layers.3.weight"], sd[p + "out_layers.3.bias"], padding=2)
            h = h + t
            i += 1
        h = F.conv1d(h, sd[f"enc.res.{i}.op.weight"], sd[f"enc.res.{i}.op.bias"], stride=4, padding=2)
        i += 1
    h = F.conv1d(F.silu(_gn(h, sd["enc.final.0.weight"], sd["enc.final.0.bias"])), sd["enc.final.2.weight"],
                 sd["enc.final.2.bias"])
    for a in range(ATTN_BLOCKS):
        h = attention_block(sd, f"enc.attn.{a}.", h, HEADS, rel_pos=False)
    return F.linear(h[:, :, 0], sd["head.weight"], sd["head.bias"])


def classify(sd, clip):
    """`classify_audio_clip`: softmax(logits)[0][0] as a 0-d tensor."""
    return F.softmax(logits(sd, clip), dim=-1)[0][0]
