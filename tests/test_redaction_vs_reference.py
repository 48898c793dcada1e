"""CPU, reference: the restatement in tortoise_tts_b200/redaction.py against the unmodified Wav2VecAlignment
(utils/wav2vec_alignment.py). The reference object is built without downloading anything: its model is a stand-in
whose forward returns given logits, its tokenizer an HF Wav2Vec2CTCTokenizer over a synthetic vocab.json."""
import json
import random

import pytest
import torch

from tortoise_tts_b200 import redaction as R
from tortoise_tts_b200.synth import W2V_VOCAB

pytestmark = pytest.mark.reference


@pytest.fixture(scope="module")
def ref():
    from oracle.ref_shims import load_reference
    load_reference()
    import tortoise.utils.wav2vec_alignment as w
    return w


class _Logits(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.next = None

    def forward(self, x):
        return type("Out", (), {"logits": self.next.unsqueeze(0)})()


@pytest.fixture(scope="module")
def aligners(ref, tmp_path_factory):
    from transformers import Wav2Vec2CTCTokenizer
    vocab = {t: i for i, t in enumerate(W2V_VOCAB)}
    p = tmp_path_factory.mktemp("tok") / "vocab.json"
    p.write_text(json.dumps(vocab))
    a = object.__new__(ref.Wav2VecAlignment)
    a.model, a.tokenizer, a.device = _Logits(), Wav2Vec2CTCTokenizer(str(p)), "cpu"
    return a, R.CTCCharTokenizer(vocab), vocab


def test_max_alignment_bit_identical(ref):
    rng = random.Random(0)
    for n in range(300):
        al = "abcde " if n % 2 else "ab"
        s1 = "".join(rng.choice(al) for _ in range(rng.randint(0, 25)))
        s2 = "".join(rng.choice(al + "xy") for _ in range(rng.randint(0, 25)))
        assert R.max_alignment(s1, s2) == ref.max_alignment(s1, s2), (s1, s2)


def _random_case(rng, vocab):
    """Logits whose argmax mostly spells a text with noise: dropped, repeated and substituted characters."""
    words = ["i", "am", "sad", "hello", "there", "feed", "me", "please", "a", "b"]
    text = " ".join(rng.choice(words) for _ in range(rng.randint(1, 6)))
    if rng.random() < 0.7:
        k = rng.randrange(len(text) + 1)
        j = rng.randrange(k, len(text) + 1)
        text = text[:k] + "[" + text[k:j] + "]" + text[j:]
    if rng.random() < 0.3:
        text = text.capitalize() + rng.choice([".", ",", "!", ""])
    bare = text.replace("[", "").replace("]", "").lower()
    ids = []
    for ch in bare:
        r = rng.random()
        if r < 0.1:
            continue
        tok = vocab.get("|" if ch == " " else ch, 3)
        if r < 0.2:
            tok = rng.randrange(len(vocab))
        ids += [tok] * rng.randint(1, 4) + [0] * rng.randint(0, 2)
    ids += [0] * rng.randint(1, 5)
    logits = torch.randn(len(ids), len(vocab))
    logits[torch.arange(len(ids)), torch.tensor(ids)] += 10.0
    return text, logits


def test_align_and_redact_bit_identical(aligners, tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)            # the reference writes alignment_debug.pth where it fails
    a, tok, vocab = aligners
    rng = random.Random(1)
    torch.manual_seed(1)
    checked = raised = 0
    for _ in range(250):
        text, logits = _random_case(rng, vocab)
        comp = rng.randint(100, 400)
        audio = torch.randn(1, logits.shape[0] * comp + rng.randint(0, comp - 1))
        ids = logits.argmax(-1).tolist()
        a.model.next = logits
        bare = text.replace("[", "").replace("]", "")
        try:
            want = a.align(audio, bare)
        except AssertionError:
            with pytest.raises(AssertionError):
                R.align(ids, audio.shape[-1], bare, tok)
            raised += 1
            continue
        # the reference resamples the audio to 16 kHz before its model; only the length enters the alignment
        assert R.align(ids, audio.shape[-1], bare, tok) == want, text
        a.model.next = logits
        try:
            w = a.redact(audio, text)
        except (AssertionError, RuntimeError, ValueError):     # every part bracketed: nothing to concatenate
            with pytest.raises((AssertionError, RuntimeError, ValueError)):
                R.redact(audio, text, ids, tok)
            continue
        assert torch.equal(R.redact(audio, text, ids, tok), w), text
        checked += 1
    assert checked >= 200, (checked, raised)
