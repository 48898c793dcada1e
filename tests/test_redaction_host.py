"""CPU: the host half of prompt redaction (tortoise_tts_b200/redaction.py) and the wav2vec2 engine's orchestration under
the torch emulation of libttb.so (tests/lib_emu.py, tests/lib_emu_wav2vec.py)."""
import json
import random

import pytest
import torch

from tortoise_tts_b200 import redaction as R
from tortoise_tts_b200.synth import synth_wav2vec, W2V_VOCAB


def _hf_tokenizer(tmp_path, vocab):
    from transformers import Wav2Vec2CTCTokenizer
    p = tmp_path / "vocab.json"
    p.write_text(json.dumps(vocab))
    return Wav2Vec2CTCTokenizer(str(p))


@pytest.fixture
def vocab():
    return {t: i for i, t in enumerate(W2V_VOCAB)}


def test_tokenizer_matches_hf(tmp_path, vocab):
    hf = _hf_tokenizer(tmp_path, vocab)
    tok = R.CTCCharTokenizer.from_path(str(tmp_path / "vocab.json"))
    rng = random.Random(0)
    alphabet = "abcdefghij ,.'~?XZ"
    for _ in range(300):
        s = "".join(rng.choice(alphabet) for _ in range(rng.randint(0, 30)))
        assert tok.encode(s) == hf.encode(s), s
        ids = [rng.randrange(len(vocab) + 3) for _ in range(rng.randint(0, 40))]
        ids += [ids[-1]] * 3 if ids else []
        assert tok.decode(ids) == hf.decode(ids), ids


def test_max_alignment_known_answers():
    assert R.max_alignment("", "abc") == ""
    assert R.max_alignment("abc", "") == "~~~"
    assert R.max_alignment("abc", "abc") == "abc"
    assert R.max_alignment("hello world", "helo wrld") == "hel~o w~rld"
    assert R.max_alignment("abc", "xbz") == "~b~"
    # tie between skipping in s1 and in s2: the reference skips the s1 character (take_s1 only when strictly better)
    assert R.max_alignment("ab", "ba") == "~b"
    with pytest.raises(AssertionError):
        R.max_alignment("a~b", "ab")


def test_max_alignment_long_text_is_iterative():
    rng = random.Random(1)
    s1 = "".join(rng.choice("abcde fgh") for _ in range(2000))
    s2 = "".join(c for c in s1 if rng.random() > 0.1)
    out = R.max_alignment(s1, s2)
    assert len(out) == 2000
    assert out.replace("~", "") == s2      # s2 is a subsequence of s1: every character of it is kept


def _spell(text, tok, frames_per_char=3, blank_gap=1):
    """argmax ids that spell `text`: char k occupies frames [k*(f+g), k*(f+g)+f), blanks in between."""
    ids = []
    starts = []
    for ch in text.lower():
        starts.append(len(ids))
        ids += tok.encode(ch) * frames_per_char + [0] * blank_gap
    return ids, starts


def test_redact_cuts_at_expected_frames(vocab):
    tok = R.CTCCharTokenizer(vocab)
    text = "[i am sad,] hi there"      # no doubled letter: a repeat would match the same run of frames twice
    bare, keep = R.split_brackets(text)
    assert bare == "i am sad, hi there" and keep == [(9, 17)]
    ids, starts = _spell(bare, tok)
    comp = 7
    audio = torch.arange(len(ids) * comp, dtype=torch.float32).reshape(1, -1)
    got = R.redact(audio, text, ids, tok)
    # character k heard at frame starts[k]; the cut keeps [start of char 9, start of char 17)
    assert torch.equal(got, audio[:, starts[9] * comp:starts[17] * comp])
    al = R.align(ids, audio.shape[-1], bare, tok)
    assert al == [0] + [s * comp for s in starts[1:]]


def test_redact_interpolates_unheard_characters(vocab):
    tok = R.CTCCharTokenizer(vocab)
    ids, starts = _spell("ab d", tok)          # the model never hears the 'c' of "abcd"
    comp = 10
    al = R.align(ids, len(ids) * comp, "abc d", tok)
    # 'c' is placed halfway between 'b' and ' '
    assert al[0] == 0 and al[1] == starts[1] * comp and al[3] == starts[2] * comp
    assert al[2] == (al[3] - al[1]) // 2 + al[1]


def test_unpaired_bracket_raises(vocab):
    tok = R.CTCCharTokenizer(vocab)
    with pytest.raises(AssertionError):
        R.redact(torch.zeros(1, 100), "[never closed", [1, 2, 3], tok)
    with pytest.raises(AssertionError):
        R.Aligner(engine=None, tokenizer=tok).redact(torch.zeros(1, 100), "ok [ then")


def test_text_without_brackets_is_untouched(vocab):
    a = torch.randn(1, 50)
    assert R.redact(a, "plain text", [], R.CTCCharTokenizer(vocab)) is a


def test_alignment_failure_raises_without_debug_file(vocab, tmp_path, monkeypatch):
    tok = R.CTCCharTokenizer(vocab)
    monkeypatch.chdir(tmp_path)
    ids, _ = _spell("ab", tok)
    # "İ".lower() is two characters: the placed characters no longer line up with the text
    with pytest.raises(AssertionError):
        R.align(ids, 80, "abİ", tok)
    assert not (tmp_path / "alignment_debug.pth").exists()


# ---------------------------------------------------------------- engine orchestration under the emulation
@pytest.fixture
def emulated_lib():
    import lib_emu_wav2vec as emu
    saved = emu.install()
    try:
        yield
    finally:
        emu.uninstall(saved)


def test_engine_orchestration_matches_hf(emulated_lib):
    from transformers import Wav2Vec2Config, Wav2Vec2ForCTC
    from tortoise_tts_b200.wav2vec_engine import Wav2VecEngine
    import torchaudio
    cfg, sd, _ = synth_wav2vec("small", seed=3)
    eng = Wav2VecEngine(cfg, sd, device="cpu")
    g = torch.Generator().manual_seed(0)
    wav = torch.randn(24000 + 371, generator=g) * 0.3       # odd lengths along the conv stack
    got = eng.logits(wav)
    m = Wav2Vec2ForCTC(Wav2Vec2Config(**cfg)).eval()
    m.load_state_dict(sd)
    with torch.no_grad():
        a = torchaudio.functional.resample(wav.reshape(1, -1), 24000, 16000)
        want = m((a - a.mean()) / torch.sqrt(a.var() + 1e-7)).logits[0]
    assert got.shape == want.shape
    err = (got - want).abs().max().item() / want.abs().max().item()
    assert err < 0.03, err
    ids = eng.ids(wav)
    assert ids.dtype == torch.int32 and torch.equal(ids.long(), got.argmax(-1))


def test_engine_rejects_other_architectures():
    from tortoise_tts_b200.wav2vec_engine import check_config
    cfg, _, _ = synth_wav2vec("small")
    check_config(cfg)
    for k, v in (("do_stable_layer_norm", False), ("feat_extract_norm", "group"), ("hidden_act", "relu"),
                 ("conv_stride", [5, 2, 2, 2, 2, 2, 1]), ("conv_bias", False)):
        with pytest.raises(ValueError, match=k.split("_")[0]):
            check_config(dict(cfg, **{k: v}))
