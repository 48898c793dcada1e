"""Prompt redaction (Tortoise's `[bracketed prompt]` feature, utils/wav2vec_alignment.py): the text between `[` and `]`
steers the delivery but is cut from the returned audio. A wav2vec2 CTC model (wav2vec_engine.Wav2VecEngine, on the
device) says which character is spoken in which frame; everything here is host string work on its argmax ids.

One deliberate difference from the reference: when the alignment fails, `align` raises AssertionError without writing
`alignment_debug.pth` into the caller's working directory.
"""
import json
import os
from itertools import groupby

import torch

SKIP = "~"


class CTCCharTokenizer:
    """Character-level CTC tokenizer over an HF `vocab.json` (what Wav2Vec2CTCTokenizer does for single-character
    vocabularies). `decode`: merge repeated ids, drop the pad (CTC blank) token, word delimiter -> space, strip.
    `encode`: space -> word delimiter, every character -> its id, unknown characters -> the unk id (None when the vocab
    has no unk token). Multi-character vocabulary entries (`<pad>`, ...) are not searched for inside the text."""

    def __init__(self, vocab, pad_token="<pad>", unk_token="<unk>", word_delimiter_token="|", do_lower_case=False,
                 clean_up_tokenization_spaces=False):
        self.vocab = dict(vocab)
        self.inv = {v: k for k, v in self.vocab.items()}
        self.pad, self.unk, self.delim = pad_token, unk_token, word_delimiter_token
        self.lower = bool(do_lower_case)
        self.clean_up = bool(clean_up_tokenization_spaces)

    @classmethod
    def from_path(cls, path):
        """`path`: a vocab.json, or a directory holding one (plus tokenizer_config.json / special_tokens_map.json,
        whose token settings are honoured)."""
        d = path if os.path.isdir(path) else os.path.dirname(path)
        vf = os.path.join(path, "vocab.json") if os.path.isdir(path) else path
        with open(vf, encoding="utf-8") as f:
            vocab = json.load(f)
        kw = {}
        for name in ("special_tokens_map.json", "tokenizer_config.json"):
            p = os.path.join(d, name)
            if os.path.exists(p):
                with open(p, encoding="utf-8") as f:
                    cfg = json.load(f)
                for k in ("pad_token", "unk_token", "word_delimiter_token", "do_lower_case",
                          "clean_up_tokenization_spaces"):
                    v = cfg.get(k)
                    if isinstance(v, dict):           # AddedToken serialisation
                        v = v.get("content")
                    if v is not None:
                        kw[k] = v
        return cls(vocab, **kw)

    def encode(self, text):
        if self.lower:
            text = text.upper()
        unk = self.vocab.get(self.unk)
        return [self.vocab.get(ch, unk) for ch in text.replace(" ", self.delim)]

    def decode(self, ids):
        toks = [self.inv.get(int(i), self.unk) for i in ids]
        chars = [" " if t == self.delim else t for t, _ in groupby(toks) if t != self.pad]
        s = "".join(chars).strip()
        if self.lower:
            s = s.lower()
        if self.clean_up:
            for a, b in ((" .", "."), (" ?", "?"), (" !", "!"), (" ,", ","), (" ' ", "'"), (" n't", "n't"),
                         (" 'm", "'m"), (" 's", "'s"), (" 've", "'ve"), (" 're", "'re")):
                s = s.replace(a, b)
        return s


def max_alignment(s1, s2, skip_character=SKIP):
    """s1 laid over s2: every character of s1 that the best alignment does not find in s2 becomes `skip_character`.

    The alignment maximises the number of kept characters (a longest common subsequence). Among equally good ones it
    makes the reference's choices: on a mismatch it skips a character of s2 only when that keeps strictly more
    characters than skipping the character of s1. Iterative (no recursion limit): a suffix-LCS table, then one walk."""
    assert skip_character not in s1, f"Found the skip character {skip_character} in the provided string, {s1}"
    import numpy as np
    n1, n2 = len(s1), len(s2)
    if n1 == 0:
        return ""
    if n2 == 0:
        return skip_character * n1
    a = np.frombuffer(s1.encode("utf-32-le"), dtype=np.uint32)
    b = np.frombuffer(s2.encode("utf-32-le"), dtype=np.uint32)
    # S[i, j] = LCS(s1[i:], s2[j:]) = max(S[i, j + 1], match ? 1 + S[i + 1, j + 1] : S[i + 1, j]): a suffix maximum
    S = np.zeros((n1 + 1, n2 + 1), dtype=np.int32)
    for i in range(n1 - 1, -1, -1):
        nxt = S[i + 1]
        m = np.where(b == a[i], nxt[1:] + 1, nxt[:-1])
        S[i, :n2] = np.maximum.accumulate(m[::-1])[::-1]
    # equal suffixes end the walk at once (s1[i:] == s2[j:] is possible on one diagonal only)
    d = n2 - n1
    out = []
    i = j = 0
    while i < n1:
        if j == n2:
            out.append(skip_character * (n1 - i))
            break
        if j - i == d and s1[i:] == s2[j:]:
            out.append(s1[i:])
            break
        if s1[i] == s2[j]:
            out.append(s1[i])
            i += 1
            j += 1
        elif S[i, j + 1] > S[i + 1, j]:
            j += 1
        else:
            out.append(skip_character)
            i += 1
    return "".join(out)


def align(ids, orig_len, expected_text, tokenizer):
    """Sample index (at the waveform's own rate) where each character of `expected_text` starts.

    ids: argmax token per model frame (sequence of ints); orig_len: waveform length, so one frame covers
    orig_len // len(ids) samples. Characters the model did not hear get positions interpolated between their heard
    neighbours. Raises AssertionError when the characters cannot be placed."""
    ids = [int(t) for t in ids]
    fixed = max_alignment(expected_text.lower(), tokenizer.decode(ids))
    per_frame = orig_len // len(ids)
    tokens = tokenizer.encode(fixed)
    if len(tokens) == 1:
        return [0]
    # the first character is placed at 0; the rest are matched in order against the frames
    want = list(zip(tokens[1:], fixed[1:]))
    pos = 0
    starts = [0]

    def next_heard():
        """Advance to the next character the alignment kept (skipped ones get -1); None when none is left."""
        nonlocal pos
        while pos < len(want):
            tok, ch = want[pos]
            pos += 1
            if ch != SKIP:
                return tok
            starts.append(-1)
        return None

    target = next_heard()
    for frame, top in enumerate(ids):
        if target is not None and target == top:
            starts.append(frame * per_frame)
            if pos == len(want):
                break
            target = next_heard()
    next_heard()
    if pos != len(want) or len(starts) != len(expected_text):
        raise AssertionError("wav2vec2 alignment failed: %d of %d characters placed for %r" %
                             (len(starts), len(expected_text), expected_text))
    # unheard characters: spread evenly between the previous placed start and the next one (or the clip's end)
    starts.append(orig_len)
    i = 0
    while i < len(starts):
        if starts[i] != -1:
            i += 1
            continue
        k = i
        while starts[k] == -1:
            k += 1
        lo, span = starts[i - 1], k - i + 1
        gap = starts[k] - lo
        for j in range(i, k):
            starts[j] = (j - i + 1) * gap // span + lo
        i = k
    return starts[:-1]


def split_brackets(text):
    """-> (bare text without brackets, [(first, last) character index of every kept segment]). Every `[` must be
    followed by a `]` (no nesting)."""
    head, *rest = text.split("[")
    parts = [head]
    for seg in rest:
        assert "]" in seg, 'Every "[" character must be paired with a "]" with no nesting.'
        parts.extend(seg.split("]"))
    keep = []
    at = 0
    for k, seg in enumerate(parts):
        if k % 2 == 0 and seg:                # even parts are spoken text; empty ones are skipped
            keep.append((at, max(0, at + len(seg) - 1)))
        at += len(seg)
    return "".join(parts), keep


def redact(audio, expected_text, ids, tokenizer):
    """audio [channels, samples]; ids: the aligner's argmax per frame for this audio. Returns audio without the
    bracketed parts of `expected_text` (`audio` itself when there are none)."""
    if "[" not in expected_text:
        return audio
    bare, keep = split_brackets(expected_text)
    starts = align(ids, audio.shape[-1], bare, tokenizer)
    return torch.cat([audio[:, starts[a]:starts[b]] for a, b in keep], dim=-1)


class Aligner:
    """Wav2VecAlignment on the device engine: `redact(audio, text)` as utils/wav2vec_alignment.py:125-150."""

    def __init__(self, engine, tokenizer):
        self.engine, self.tokenizer = engine, tokenizer

    def redact(self, audio, expected_text):
        """audio [1, samples] at 24 kHz on the device."""
        if "[" not in expected_text:
            return audio
        split_brackets(expected_text)              # unpaired brackets fail before the model runs
        ids = self.engine.ids(audio).cpu().tolist()
        return redact(audio, expected_text, ids, self.tokenizer)
