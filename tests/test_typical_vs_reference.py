"""The typical-sampling oracle (tests/typical_oracle.py) against the reference's own TypicalLogitsWarper
(tortoise/utils/typical_sampling.py) inside the HF processor chain of the installed transformers: RepetitionPenalty ->
TypicalLogitsWarper -> Temperature -> TopK -> TopP (stream_generator.py:946-947, autoregressive.py:558)."""
import pytest
import torch

import typical_oracle

pytestmark = pytest.mark.reference


def _chain(logits, prev, mass, temperature=0.8, top_k=50, top_p=0.8):
    from oracle.ref_shims import load_reference
    load_reference()
    from tortoise.utils.typical_sampling import TypicalLogitsWarper
    from transformers.generation.logits_process import (RepetitionPenaltyLogitsProcessor, TemperatureLogitsWarper,
                                                        TopKLogitsWarper, TopPLogitsWarper)
    s = RepetitionPenaltyLogitsProcessor(2.0)(prev, logits.clone())
    s = TypicalLogitsWarper(mass=mass)(prev, s)
    s = TemperatureLogitsWarper(temperature)(prev, s)
    s = TopKLogitsWarper(top_k)(prev, s)
    s = TopPLogitsWarper(top_p)(prev, s)
    return torch.softmax(s, dim=-1)[0]


def _check(logits, prev, mass, **kw):
    p = _chain(logits, prev, mass, **kw)
    tok, kept, kp = typical_oracle.sample_step(logits[0], prev[0].tolist(), 0.5, typical_mass=mass, **kw)
    ref_kept = (p > 0).nonzero().flatten()
    assert sorted(kept.tolist()) == sorted(ref_kept.tolist())
    assert (p[kept] - kp).abs().max().item() < 1e-6
    assert tok in kept.tolist()
    return kept


def _prev(g, n=20):
    return torch.cat([torch.tensor([[1] * 10 + [8192]]), torch.randint(0, 8192, (1, n), generator=g)], dim=1)


@pytest.mark.parametrize("mass", [0.2, 0.5, 0.9, 0.999])
@pytest.mark.parametrize("scale", [0.5, 3.0, 10.0])
def test_random_logits(mass, scale):
    g = torch.Generator().manual_seed(int(mass * 1000) + int(scale * 10))
    for _ in range(3):
        _check(torch.randn(1, 8194, generator=g) * scale, _prev(g), mass)


def test_typical_set_smaller_than_top_k():
    """|T| < top_k: top-k must not pull masked tokens back in."""
    g = torch.Generator().manual_seed(11)
    logits = torch.randn(1, 8194, generator=g) * 0.1
    logits[0, :5] = torch.tensor([20.0, 19.8, 19.6, 19.4, 19.2])
    for mass in (0.2, 0.5, 0.9):
        keep, _ = typical_oracle.typical_keep(logits[0], mass)
        assert 1 < int(keep.sum()) < 50
        _check(logits, _prev(g), mass, top_p=1.0)


def test_single_token_set():
    g = torch.Generator().manual_seed(12)
    logits = torch.randn(1, 8194, generator=g)
    logits[0, 777] = 40.0
    keep, _ = typical_oracle.typical_keep(logits[0], 0.5)
    assert int(keep.sum()) == 1
    assert _check(logits, _prev(g), 0.5).tolist() == [777]


def test_ties_at_the_threshold():
    """Rows made of a few levels of exactly equal logits: every key ties with a whole level, so v always sits on a tie
    and every token tied with v must be kept whatever the sort order. Compared at the output of the warper (a top-k over
    such rows keeps every tie of its k-th value in HF, which is not the typical filter's business)."""
    from oracle.ref_shims import load_reference
    load_reference()
    from tortoise.utils.typical_sampling import TypicalLogitsWarper
    g = torch.Generator().manual_seed(13)
    for levels in ([2.0, 0.0], [1.0, 0.5, -3.0], [0.0], [4.0, 1.0, 0.0, -1.0]):
        logits = torch.tensor(levels)[torch.randint(0, len(levels), (1, 8194), generator=g)]
        for mass in (0.2, 0.5, 0.9, 0.999):
            want = torch.isfinite(TypicalLogitsWarper(mass=mass)(None, logits.clone()))[0]
            keep, v = typical_oracle.typical_keep(logits[0], mass)
            assert torch.equal(keep, want)
            assert int(keep.sum()) >= 2


def test_penalised_ids():
    g = torch.Generator().manual_seed(14)
    logits = torch.randn(1, 8194, generator=g) * 2
    prev = torch.cat([torch.tensor([[1, 8192]]), logits[0].topk(30).indices.unsqueeze(0)], dim=1)
    logits[0, prev[0, 2:12]] *= -1.0
    for mass in (0.2, 0.5, 0.9, 0.999):
        _check(logits, prev, mass)
