"""Drop-in facade for `tortoise.api_fast.TextToSpeech` (tortoise/api_fast.py:171-520) on the sm_90a engine: the
reference's low-latency product path — ONE autoregressive sequence, no CLVP / diffusion, GPT latents rendered
directly by the HiFiGAN decoder (`hifidecoder.pth`), optionally streamed chunk by chunk.

Same constructor, `tts()`, `tts_stream()`, `tts_with_preset()`, `handle_chunks()`, `get_conditioning_latents()`
(auto latent only, api_fast.py:225-246), `get_random_conditioning_latents()` (api_fast.py:248-254) and
`deterministic_state()`. Beyond the reference: `tts_batch()` / `tts_long()` (many sentences in one decode batch) and
their streaming forms `tts_stream_batch()` / `tts_long_stream()`, and `stream_pool()` (texts that arrive while
others stream join the running decode batch). Everything between the tokenizer and the returned waveform runs in libttb.so: the decode
loop (`AREngine.generate` / `generate_stream`), the latent pass (`AREngine.latents` / `stream_latents`) and the
decoder (`HifiganEngine`).

Deliberate differences (SURVEY App. D): sampling randomness comes from a device generator seeded by
`use_deterministic_seed`; `tts_with_preset` drops the diffusion-only preset keys instead of forwarding them to HF
`generate` (which rejects them in the reference); the wav2vec redaction model is not loaded.
"""
import collections
import os
import random
import threading
from time import perf_counter, time

import torch

from .config import ModelConfig
from .ar_engine import AREngine
from .conditioning_engine import ConditioningEngine, RandomLatentEngine
from .hifigan_engine import HifiganEngine
from . import lib
from . import parallel
from .api import MODELS_DIR, _Tokenizer, _default_mel_norms, _typical_mass
# module-level names callers of tortoise/api_fast.py import from it (api_fast.py:52-171)
from .api import pad_or_truncate, format_conditioning, pick_best_batch_size_for_gpu, classify_audio_clip  # noqa: F401

MODELS = ("autoregressive.pth", "classifier.pth", "clvp2.pth", "cvvp.pth", "diffusion_decoder.pth", "vocoder.pth",
          "rlg_auto.pth", "rlg_diffuser.pth", "hifidecoder.pth")       # api_fast.py:31-43

PRESETS = {  # api_fast.py:265-270
    "ultra_fast": {"num_autoregressive_samples": 1, "diffusion_iterations": 10},
    "fast": {"num_autoregressive_samples": 32, "diffusion_iterations": 50},
    "standard": {"num_autoregressive_samples": 256, "diffusion_iterations": 200},
    "high_quality": {"num_autoregressive_samples": 256, "diffusion_iterations": 400},
}
_DIFFUSION_ONLY = ("diffusion_iterations", "cond_free", "cond_free_k", "diffusion_temperature")
STREAM_MAX_LENGTH = 500      # autoregressive.py:571: prompt + generated tokens of the streaming generator
FIRST_BUFFER = 60            # api_fast.py:398
POOL_ADMIT_STEPS = 16        # StreamPool: decode steps between two looks at its queue


def stream_flushes(n, flushed, ended, stream_chunk_size):
    """The flush rule of the streaming mode (api_fast.py:393-419), for one stream: `n` tokens have arrived, the previous
    flush covered `flushed` of them (0: none yet), `ended` says whether the stream is over. Returns the flushes due now,
    in order, as a list of `is_end` flags: one flush when the tokens buffered since the last flush reach the threshold
    (max(stream_chunk_size, 60) before the first flush, stream_chunk_size after it; never when stream_chunk_size <= 0),
    and one more when the stream has ended, even if nothing arrived since the last flush."""
    every = int(stream_chunk_size)
    due = every > 0 and (n - flushed) >= (max(every, FIRST_BUFFER) if flushed == 0 else every)
    return ([False] if due else []) + ([True] if ended else [])


STREAM_SETTINGS = ("temperature", "top_p", "top_k", "repetition_penalty", "length_penalty")   # per stream / per text
BATCH_SETTINGS = STREAM_SETTINGS + ("typical_sampling", "typical_mass")                      # per sentence of tts_batch


def row_settings(kwargs_list, n, base, allowed):
    """The per-text sampling settings of a batch: `kwargs_list` (one dict per text, keys from `allowed`) over `base` (the
    call's own settings, a dict with every key of `allowed`), validated before any work starts: a list whose length is
    not n raises ValueError, a key outside `allowed` TypeError, a bad value ValueError (lib.sample_params_row). Returns
    one dict per text for the engine (temperature, top_k, top_p, repetition_penalty, typical_mass);
    length_penalty is accepted and has no effect, as in tts_stream."""
    kwargs_list = list(kwargs_list)
    if len(kwargs_list) != n:
        raise ValueError("kwargs_list has %d entries for %d texts" % (len(kwargs_list), n))
    out = []
    for u, kw in enumerate(kwargs_list):
        unknown = set(kw) - set(allowed)
        if unknown:
            raise TypeError("kwargs_list[%d]: unsupported settings %s" % (u, sorted(unknown)))
        m = {**base, **kw}
        row = dict(temperature=m["temperature"], top_k=m["top_k"], top_p=m["top_p"],
                   repetition_penalty=m["repetition_penalty"],
                   typical_mass=_typical_mass(m["typical_sampling"], m["typical_mass"]) if "typical_sampling" in m
                   else None)
        lib.sample_params_row(**row)
        out.append(row)
    return out


def get_model_path(model_name, models_dir=MODELS_DIR):
    if model_name not in MODELS:
        raise ValueError(f"Model {model_name} not found in available models.")
    path = os.path.join(models_dir, model_name)
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path} missing (this build is offline: place the reference checkpoints there)")
    return path


class TextToSpeech:
    def __init__(self, autoregressive_batch_size=None, models_dir=MODELS_DIR, enable_redaction=True, kv_cache=False,
                 use_deepspeed=False, half=False, device=None, tokenizer_vocab_file=None, tokenizer_basic=False,
                 state_dicts=None, config: ModelConfig = None):
        """`state_dicts` (keys autoregressive / hifigan [/ rlg_auto / mel_norms]) bypasses models_dir (synthetic
        checkpoints); `config` overrides the full-size ModelConfig (tests)."""
        if not torch.cuda.is_available():
            raise RuntimeError("tortoise_tts_b200 needs a CUDA device (sm_90a); there is no CPU path")
        lib.load()
        self.models_dir = models_dir
        self.autoregressive_batch_size = autoregressive_batch_size     # accepted for API parity (one sequence is decoded)
        self.enable_redaction = False       # wav2vec redaction is out of scope (SURVEY §2 #15)
        self.kv_cache = kv_cache
        self.half = half
        self.device = torch.device(device if device is not None else "cuda")
        if self.device.type == "cuda":
            torch.cuda.set_device(self.device if self.device.index is not None else torch.cuda.current_device())
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.cfg = config or ModelConfig.full()
        self._tok_file, self._tok_basic, self._tokenizer = tokenizer_vocab_file, bool(tokenizer_basic), None
        if state_dicts is None:
            state_dicts = {
                "autoregressive": torch.load(get_model_path("autoregressive.pth", models_dir), map_location="cpu"),
                "hifigan": torch.load(get_model_path("hifidecoder.pth", models_dir), map_location="cpu"),
            }
        self._sds = state_dicts
        self.autoregressive = AREngine(state_dicts["autoregressive"], self.cfg, self.device)
        self.hifi_decoder = HifiganEngine(state_dicts["hifigan"], self.cfg, self.device)
        self._conditioning = None           # the conditioning front-end is only built when voice samples are given
        self.rlg_auto = None
        self.last_timings = {}

    # ------------------------------------------------------------------ conditioning (api_fast.py:225-254)
    def get_conditioning_latents(self, voice_samples, return_mels=False):
        """List of reference clips (22.05 kHz waveforms [1, n]) -> autoregressive conditioning latent [1, D]; the
        reference returns the same tensor with and without `return_mels` (api_fast.py:243-246)."""
        if not isinstance(voice_samples, (list, tuple)):
            voice_samples = [voice_samples]
        if self._conditioning is None:
            mn = self._sds.get("mel_norms", None)
            self._conditioning = ConditioningEngine(self._sds["autoregressive"], None, self.cfg, self.device,
                                                    mel_norms=mn if mn is not None else _default_mel_norms())
        with torch.no_grad():
            return self._conditioning.ar_latent(list(voice_samples))

    def get_random_conditioning_latents(self):
        if self.rlg_auto is None:
            sa = self._sds.get("rlg_auto")
            if sa is None:
                sa = torch.load(get_model_path("rlg_auto.pth", self.models_dir), map_location="cpu")
            self.rlg_auto = RandomLatentEngine(sa, self.cfg.ar_dim, self.device)
        with torch.no_grad():
            return self.rlg_auto()

    @property
    def tokenizer(self):
        if self._tokenizer is None:
            self._tokenizer = _Tokenizer(self._tok_file, self._tok_basic)
        return self._tokenizer

    def deterministic_state(self, seed=None):
        if seed is None:
            seed = parallel.broadcast_seed(int(time()), self.device)
        torch.manual_seed(seed)
        random.seed(seed)
        return seed

    def tts_with_preset(self, text, preset="fast", **kwargs):
        """≙ api_fast.py:256-275: a generator over the result of `tts` (the rows of the waveform tensor)."""
        settings = {"temperature": .8, "length_penalty": 1.0, "repetition_penalty": 2.0, "top_p": .8}
        settings.update({k: v for k, v in PRESETS[preset].items() if k not in _DIFFUSION_ONLY})
        settings.update({k: v for k, v in kwargs.items() if k not in _DIFFUSION_ONLY})
        for audio_frame in self.tts(text, **settings):
            yield audio_frame

    # ------------------------------------------------------------------ streaming helpers
    def handle_chunks(self, wav_gen, wav_gen_prev, wav_overlap, overlap_len):
        """Chunk formatting of the streaming mode, same results as api_fast.py:277-303: every call receives the decoder
        output for ALL latents so far; the new samples (minus a tail of `overlap_len` kept back) are returned, their head
        cross-faded linearly with the tail kept back by the previous call. Returns (chunk, wav_gen, tail)."""
        start = 0 if wav_gen_prev is None else wav_gen_prev.shape[0] - overlap_len
        chunk = wav_gen[start:-overlap_len]
        if wav_overlap is not None:
            if overlap_len > len(chunk):
                # fewer new samples than the cross-fade needs (the last chunk): hand out everything that is left
                chunk = wav_gen[start:] if wav_gen_prev is not None else wav_gen[-overlap_len:]
                return chunk, wav_gen, None
            up = torch.linspace(0.0, 1.0, overlap_len).to(chunk.device)
            down = torch.linspace(1.0, 0.0, overlap_len).to(wav_overlap.device)
            # the chunk is a view of wav_gen: the fade is written in place, as in the reference
            chunk[:overlap_len] = wav_overlap * down + chunk[:overlap_len] * up
        return chunk, wav_gen, wav_gen[-overlap_len:]

    def _inputs(self, text, voice_samples, text_tokens, use_deterministic_seed):
        seed = self.deterministic_state(seed=use_deterministic_seed)
        toks = self._inputs_tokens(text, text_tokens)
        return seed, toks, self._auto_latent(voice_samples)

    def _auto_latent(self, voice_samples):
        if voice_samples is not None:
            auto = self.get_conditioning_latents(voice_samples, return_mels=False)
        else:
            auto = self.get_random_conditioning_latents()
        return auto.to(self.device).float().reshape(-1)

    def _inputs_tokens(self, text, text_tokens):
        if text_tokens is None:
            text_tokens = self.tokenizer.encode(text)
        toks = [int(t) for t in text_tokens] + [0]            # F.pad(text_tokens, (0, 1))
        assert len(toks) < 400, "Too much text provided. Break the text up into separate segments and re-try inference."
        return toks

    def _pos_mode(self):
        return "ref_kv_quirk" if self.kv_cache else "train_consistent"

    def tts_stream(self, text, voice_samples=None, conditioning_latents=None, k=1, verbose=True,
                   use_deterministic_seed=None, return_deterministic_state=False, overlap_wav_len=1024,
                   stream_chunk_size=40, num_autoregressive_samples=512, temperature=.8, length_penalty=1,
                   repetition_penalty=2.0, top_p=.8, max_mel_tokens=500, cvvp_amount=.0, diffusion_iterations=100,
                   cond_free=True, cond_free_k=2, diffusion_temperature=1.0, text_tokens=None, top_k=50,
                   **hf_generate_kwargs):
        """≙ api_fast.py:306-420: a generator of waveform chunks (1-D fp32 tensors on the device, 24 kHz). The token
        stream is buffered until `max(stream_chunk_size, 60)` tokens have arrived, then flushed every
        `stream_chunk_size` tokens and at its end; at every flush ALL latents so far are decoded and `handle_chunks`
        cuts the new part. `conditioning_latents`, `k` and the diffusion / CVVP knobs are ignored, as in the reference."""
        if hf_generate_kwargs:
            raise TypeError(f"unsupported generate kwargs: {sorted(hf_generate_kwargs)}")
        seed, toks, auto = self._inputs(text, voice_samples, text_tokens, use_deterministic_seed)
        if verbose:
            print("Generating autoregressive samples..")
        P = len(toks) + 4                                        # fake inputs incl. the start mel token
        n_max = STREAM_MAX_LENGTH - P
        assert n_max > 0, "prompt longer than the streaming generator's max_length"
        flush_every = int(stream_chunk_size)
        first = max(flush_every, FIRST_BUFFER) if flush_every > 0 else n_max
        pos = self._pos_mode()
        with torch.no_grad():
            g = torch.Generator(device=self.device)
            g.manual_seed(seed)
            uniforms = torch.rand(1, n_max, generator=g, device=self.device)
            wav_prev = wav_tail = None
            flushed = 0                                          # tokens covered by the previous flush
            for codes, ended in self.autoregressive.generate_stream(
                    auto, toks, n_max, first, flush_every if flush_every > 0 else n_max, uniforms=uniforms,
                    temperature=temperature, top_k=top_k, top_p=top_p, repetition_penalty=repetition_penalty,
                    pos_mode=pos, use_graph=self.device.type == "cuda"):
                n = int(codes.numel())
                for is_end in stream_flushes(n, flushed, ended, flush_every):
                    lat = self.autoregressive.stream_latents(auto, toks, codes) if pos == "ref_kv_quirk" else \
                        self._stream_latents_train(auto, toks, codes)
                    wav_gen = self.hifi_decoder.inference(lat, auto)
                    chunk, wav_prev, wav_tail = self.handle_chunks(wav_gen, wav_prev, wav_tail, overlap_wav_len)
                    flushed = n
                    yield chunk

    def _stream_latents_train(self, auto, toks, codes):
        """Stream latents under the full-recompute position rule (kv_cache=False): row i of the teacher-forced latent
        pass over [start, c_0 .. c_{n-2}, c_{n-1}] (positions 0..n) is the latent that sampled c_i."""
        return self.autoregressive.latents(auto, toks, codes.reshape(1, -1))[0]

    def tts(self, text, voice_samples=None, k=1, verbose=True, use_deterministic_seed=None,
            num_autoregressive_samples=512, temperature=.8, length_penalty=1, repetition_penalty=2.0, top_p=.8,
            max_mel_tokens=500, cvvp_amount=.0, text_tokens=None, top_k=50, typical_sampling=False, typical_mass=.9,
            **hf_generate_kwargs):
        """≙ api_fast.py:421-507: ONE sampled sequence (`num_return_sequences=1`; the generation limit is the model's
        `max_mel_tokens - 1`, the `max_mel_tokens` argument is not used by the reference either) -> latents of
        `UnifiedVoice.forward(return_latent=True)` over the raw codes (stop token included, no `fix_autoregressive_output`)
        -> HiFiGAN. Returns fp32 [1, 1, samples] on the device. `typical_sampling` / `typical_mass`: as in api.tts
        (api_fast.py:484-495 passes them to the generator the same way)."""
        if hf_generate_kwargs:
            raise TypeError(f"unsupported generate kwargs: {sorted(hf_generate_kwargs)}")
        typical = _typical_mass(typical_sampling, typical_mass)
        seed, toks, auto = self._inputs(text, voice_samples, text_tokens, use_deterministic_seed)
        if verbose:
            print("Generating autoregressive samples..")
        n_max = self.cfg.max_mel_tokens - 1                      # autoregressive.py:553: trunc_index + max_mel_tokens - 1
        timed = self.device.type == "cuda"
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)] if timed else None
        mark = (lambda i: ev[i].record()) if timed else (lambda i: None)
        with torch.no_grad():
            mark(0)
            uniforms = self._uniforms(seed, n_max)
            codes = self.autoregressive.generate(auto, toks, 1, n_max, uniforms=uniforms, temperature=temperature,
                                                 top_k=top_k, top_p=top_p, repetition_penalty=repetition_penalty,
                                                 pos_mode=self._pos_mode(), use_graph=self.device.type == "cuda",
                                                 typical_mass=typical)
            wav, n = self._render(auto, toks, codes, n_max, verbose, mark, 1)
        self.last_timings = {"tokens": n}
        if timed:
            torch.cuda.synchronize()
            self.last_timings = {"ar_ms": ev[0].elapsed_time(ev[1]), "latents_ms": ev[1].elapsed_time(ev[2]),
                             "hifigan_ms": ev[2].elapsed_time(ev[3]), "tokens": n}
        return wav

    def _uniforms(self, seed, n_max):
        """The sampling randomness of one sequence: the first row of a device generator seeded with `seed`."""
        g = torch.Generator(device=self.device)
        g.manual_seed(seed)
        return torch.rand(1, n_max, generator=g, device=self.device)

    def _render(self, auto, toks, codes, n_max, verbose, mark, m0):
        """What tts() does after the decode, for one sequence `codes` [1, n_max]: cut after the first stop token (HF
        returns the stop token it sampled), latents over the raw codes, HiFiGAN. `mark(i)` (if given) records event m0
        after the cut, m0 + 1 after the latents, m0 + 2 after HiFiGAN. Returns (fp32 [1, 1, samples], tokens kept)."""
        mark = mark or (lambda i: None)
        hit = (codes[0] == self.cfg.stop_mel_token).nonzero()
        n = int(hit[0].item()) + 1 if hit.numel() > 0 else n_max
        mark(m0)
        if verbose:
            print("generating audio..")
        lat = self.autoregressive.latents(auto, toks, codes[:, :n].contiguous())[0]
        mark(m0 + 1)
        wav = self.hifi_decoder.inference(lat, auto)
        mark(m0 + 2)
        return wav.reshape(1, 1, -1), n

    # ------------------------------------------------------------------ several sentences per call
    def tts_batch(self, texts, voice_samples=None, text_tokens_list=None, conditioning_latents_list=None, kwargs_list=None,
                  **kwargs):
        """Several sentences in one call, each ONE sequence: entry u of the returned list is what
        `tts(texts[u], voice_samples, **kwargs)` returns (fp32 [1, 1, samples] on the device). The conditioning latent
        and the seed are computed once, and every sentence samples with the uniforms row tts() draws from that seed.
        The sentences are decoded together: consecutive sentences are packed into decode batches of up to 256 rows,
        one row per sentence, each attending to its own prompt (ar_engine.plan_batches), so a batch costs about one
        decode step per token instead of one per sentence and token. A sentence whose prompt is longer than 352
        positions is decoded alone, as tts() decodes it. The stop-token cut, the latent pass and HiFiGAN then run per
        sentence as in tts(). `text_tokens_list` (one id list per text) bypasses the tokenizer.
        `conditioning_latents_list`: one auto conditioning latent per text (as get_conditioning_latents returns it), so
        that one batch holds several voices; with get_conditioning_latents(clips) as entry u, entry u of the result is
        tts(texts[u], voice_samples=clips). It excludes `voice_samples`. `last_timings`: ar_ms
        (the decode batches, prefills included), prefill_ms (their prompt prefills), latents_ms and hifigan_ms (summed
        over the sentences), device_total_ms, and tokens (the tokens kept per sentence). Every rank computes the whole
        batch, as tts() does.
        `kwargs_list`: one dict per text of sampling settings (temperature, top_p, top_k, repetition_penalty,
        length_penalty, typical_sampling, typical_mass) over `kwargs`: entry u is then
        `tts(texts[u], ..., **{**kwargs, **kwargs_list[u]})`. The rows of one decode batch sample with their own settings
        (the per-row sampler); without kwargs_list every row shares the call's settings."""
        texts = list(texts)
        if not texts:
            raise ValueError("tts_batch needs at least one text")
        self._check_lists(texts, voice_samples, text_tokens_list, conditioning_latents_list)
        return self._tts_batch(texts, voice_samples, text_tokens_list, conditioning_latents_list, kwargs_list, **kwargs)

    @staticmethod
    def _check_lists(texts, voice_samples, text_tokens_list, conditioning_latents_list):
        if text_tokens_list is not None and len(text_tokens_list) != len(texts):
            raise ValueError("text_tokens_list has %d entries for %d texts" % (len(text_tokens_list), len(texts)))
        if conditioning_latents_list is not None:
            if voice_samples is not None:
                raise ValueError("give voice_samples (one voice for every text) or conditioning_latents_list, not both")
            if len(conditioning_latents_list) != len(texts):
                raise ValueError("conditioning_latents_list has %d entries for %d texts" %
                                 (len(conditioning_latents_list), len(texts)))

    def _auto_latents(self, n, voice_samples, conditioning_latents_list):
        """The auto conditioning latent of each of n texts: conditioning_latents_list, else one voice for all."""
        if conditioning_latents_list is not None:
            return [c.to(self.device).float().reshape(-1) for c in conditioning_latents_list]
        return [self._auto_latent(voice_samples)] * n

    def _tts_batch(self, texts, voice_samples, text_tokens_list, conditioning_latents_list, kwargs_list, k=1, verbose=True,
                   use_deterministic_seed=None,
                   num_autoregressive_samples=512, temperature=.8, length_penalty=1, repetition_penalty=2.0, top_p=.8,
                   max_mel_tokens=500, cvvp_amount=.0, top_k=50, typical_sampling=False, typical_mass=.9,
                   **hf_generate_kwargs):
        from .ar_engine import plan_batches
        if hf_generate_kwargs:
            raise TypeError(f"unsupported generate kwargs: {sorted(hf_generate_kwargs)}")
        typical = _typical_mass(typical_sampling, typical_mass)
        settings = None if kwargs_list is None else row_settings(
            kwargs_list, len(texts), dict(temperature=temperature, top_k=top_k, top_p=top_p,
                                          repetition_penalty=repetition_penalty, length_penalty=length_penalty,
                                          typical_sampling=typical_sampling, typical_mass=typical_mass), BATCH_SETTINGS)
        seed = self.deterministic_state(seed=use_deterministic_seed)
        toks = [self._inputs_tokens(texts[u], None if text_tokens_list is None else text_tokens_list[u])
                for u in range(len(texts))]
        autos = self._auto_latents(len(texts), voice_samples, conditioning_latents_list)
        if verbose:
            print("Generating autoregressive samples..")
        n_max = self.cfg.max_mel_tokens - 1
        ar = self.autoregressive
        timed = self.device.type == "cuda"
        dec = dict(temperature=temperature, top_k=top_k, top_p=top_p, repetition_penalty=repetition_penalty,
                   pos_mode=self._pos_mode(), use_graph=timed, typical_mass=typical)
        new_events = (lambda n: [torch.cuda.Event(enable_timing=True) for _ in range(n)]) if timed else \
            (lambda n: None)
        sums = {"ar_ms": 0.0, "prefill_ms": 0.0, "latents_ms": 0.0, "hifigan_ms": 0.0}
        timed_parts = []                                         # (events, [(key, i, j), ...]) read after one sync
        wavs, tokens = [None] * len(texts), [0] * len(texts)
        ends = new_events(2)
        with torch.no_grad():
            if timed:
                ends[0].record()
            uniforms = self._uniforms(seed, n_max)
            # the grouped step needs the one-kernel step; with the per-op step forced every sentence decodes alone
            max_groups = 1 if ar.MODE == "perop" else lib.AR_STEP_MAX_GROUPS
            for batch in plan_batches([(1, len(t) + 4) for t in toks], max_groups=max_groups):
                ev = new_events(4)                               # decode start, prefills start / end, decode end
                pre = (ev[1], ev[2]) if timed else None
                if timed:
                    ev[0].record()
                if len(batch) == 1:
                    one = dec if settings is None else {**dec, **settings[batch[0]]}
                    codes = [ar.generate(autos[batch[0]], toks[batch[0]], 1, n_max, uniforms=uniforms,
                                         prefill_events=pre, **one)]
                else:
                    per_row = {} if settings is None else {"row_settings": [settings[u] for u in batch]}
                    codes = ar.generate_grouped([autos[u] for u in batch], [toks[u] for u in batch], [1] * len(batch),
                                                n_max, uniforms_list=[uniforms] * len(batch), prefill_events=pre,
                                                **dec, **per_row)
                if timed:
                    ev[3].record()
                    timed_parts.append((ev, [("ar_ms", 0, 3), ("prefill_ms", 1, 2)]))
                for u, c in zip(batch, codes):
                    e = new_events(3)
                    wavs[u], tokens[u] = self._render(autos[u], toks[u], c, n_max, False,
                                                      (lambda i, e=e: e[i].record()) if timed else None, 0)
                    if timed:
                        timed_parts.append((e, [("latents_ms", 0, 1), ("hifigan_ms", 1, 2)]))
            if timed:
                ends[1].record()
        self.last_timings = {"tokens": tokens}
        if timed:
            ends[1].synchronize()
            for ev, keys in timed_parts:
                for key, i, j in keys:
                    sums[key] += ev[i].elapsed_time(ev[j])
            self.last_timings = {**sums, "device_total_ms": ends[0].elapsed_time(ends[1]), "tokens": tokens}
        return wavs

    def tts_long(self, text, text_tokens_list=None, **kwargs):
        """≙ the loop of the reference's `read_fast.py:44-76` for one voice: split the text (`'|'` forces the split
        points, else `split_and_recombine_text`), render every chunk with the SAME seed and conditioning latent (one
        tts_batch call), and concatenate the waveforms. Returns `[1, samples]` on the CPU. `text_tokens_list` (one id
        list per chunk) bypasses the tokenizer; the other keyword arguments are those of tts()."""
        from .text import split_and_recombine_text
        texts = text.split("|") if "|" in text else split_and_recombine_text(text)      # read_fast.py:45-51
        if text_tokens_list is not None and len(text_tokens_list) != len(texts):
            raise ValueError("text_tokens_list has %d entries for %d chunks" % (len(text_tokens_list), len(texts)))
        wavs = self.tts_batch(texts, text_tokens_list=text_tokens_list, **kwargs)
        return torch.cat([w.reshape(1, -1).cpu() for w in wavs], dim=-1)

    # ------------------------------------------------------------------ many streams per call
    def tts_stream_batch(self, texts, voice_samples=None, conditioning_latents_list=None, text_tokens_list=None,
                         kwargs_list=None, **kwargs):
        """Streams several texts at once: a generator of `(u, chunk, last)`. For each u, the chunks arrive in the order
        `tts_stream(texts[u], ...)` yields them, with the same count and lengths; `last` marks the final chunk of stream
        u. Chunks of different streams interleave. Every text is one row of ONE grouped decode batch (at most
        lib.AR_STEP_MAX_GROUPS texts, each prompt at most lib.AR_STEP_MAX_P positions; beyond that ValueError, since a
        stream cannot wait for another batch), so the batch costs about one decode step per token for all streams.
        Each row keeps tts_stream's flush rule (stream_flushes) and chunk state. The latents come from the decode steps
        themselves (AREngine.generate_grouped_stream) instead of a teacher-forced pass per flush, and the rows that
        flush at the same token count are decoded by one HifiganEngine.inference_batch call. The captured latents
        differ from tts_stream's recomputed ones in the last bits, so the tokens are identical and the waveforms agree
        within rounding (DESIGN §5).
        One seed for all rows: row u samples with the uniforms tts_stream draws from it for texts[u].
        `voice_samples`: one voice for all texts; `conditioning_latents_list`: one auto conditioning latent per text (as
        get_conditioning_latents returns it), not both. `text_tokens_list` (one id list per text) bypasses the
        tokenizer. The other keyword arguments are those of tts_stream, accepted and rejected as it does.
        `kwargs_list`: one dict per text of temperature / top_p / top_k / repetition_penalty / length_penalty over the
        other keyword arguments (another key raises TypeError): stream u is then that of `tts_stream(texts[u], ...,
        **{**kwargs, **kwargs_list[u]})`, each row sampling with its own settings. The chunk size stays one for the batch.
        `last_timings` (set when the generator is exhausted): ar_ms (decode, prefills included), hifigan_ms,
        device_total_ms and tokens (per row)."""
        texts = list(texts)
        if not texts:
            raise ValueError("tts_stream_batch needs at least one text")
        if len(texts) > lib.AR_STEP_MAX_GROUPS:
            raise ValueError("tts_stream_batch streams at most %d texts at once, got %d" %
                             (lib.AR_STEP_MAX_GROUPS, len(texts)))
        self._check_lists(texts, voice_samples, text_tokens_list, conditioning_latents_list)
        toks = [self._inputs_tokens(texts[u], None if text_tokens_list is None else text_tokens_list[u])
                for u in range(len(texts))]
        for u, t in enumerate(toks):
            if len(t) + 4 > lib.AR_STEP_MAX_P:
                raise ValueError("text %d: a prompt of %d positions (at most %d in a batch; tts_stream streams it alone)"
                                 % (u, len(t) + 4, lib.AR_STEP_MAX_P))
        return self._stream_batch(toks, voice_samples, conditioning_latents_list, kwargs_list, **kwargs)

    def _stream_batch(self, toks, voice_samples, conditioning_latents_list, kwargs_list, conditioning_latents=None, k=1,
                      verbose=True, use_deterministic_seed=None, return_deterministic_state=False, overlap_wav_len=1024,
                      stream_chunk_size=40, num_autoregressive_samples=512, temperature=.8, length_penalty=1,
                      repetition_penalty=2.0, top_p=.8, max_mel_tokens=500, cvvp_amount=.0, diffusion_iterations=100,
                      cond_free=True, cond_free_k=2, diffusion_temperature=1.0, top_k=50, **hf_generate_kwargs):
        """tts_stream's keyword arguments, checked before the generator starts."""
        if hf_generate_kwargs:
            raise TypeError(f"unsupported generate kwargs: {sorted(hf_generate_kwargs)}")
        dec = dict(temperature=temperature, top_k=top_k, top_p=top_p, repetition_penalty=repetition_penalty)
        if kwargs_list is not None:
            dec["row_settings"] = row_settings(kwargs_list, len(toks), dict(dec, length_penalty=length_penalty),
                                               STREAM_SETTINGS)
        return self._stream_batch_run(toks, voice_samples, conditioning_latents_list, verbose, use_deterministic_seed,
                                      overlap_wav_len, int(stream_chunk_size), dec)

    def _stream_batch_run(self, toks, voice_samples, conditioning_latents_list, verbose, use_deterministic_seed,
                          overlap_wav_len, flush_every, dec):
        R = len(toks)
        seed = self.deterministic_state(seed=use_deterministic_seed)
        autos = self._auto_latents(R, voice_samples, conditioning_latents_list)
        if verbose:
            print("Generating autoregressive samples..")
        caps = [STREAM_MAX_LENGTH - (len(t) + 4) for t in toks]
        if flush_every > 0:
            first, block = max(flush_every, FIRST_BUFFER), flush_every
        else:
            first = block = max(caps)
        timed = self.device.type == "cuda"
        new_event = (lambda: torch.cuda.Event(enable_timing=True)) if timed else (lambda: None)
        record = (lambda e: e.record()) if timed else (lambda e: None)
        ar_parts, hifi_parts = [], []
        wav_prev, wav_tail, flushed = [None] * R, [None] * R, [0] * R
        done, tokens = [False] * R, [0] * R
        with torch.no_grad():
            start = new_event()
            record(start)
            # as tts_stream: each row draws its own table from the seed (a Philox draw depends on the tensor's size)
            us = [self._uniforms(seed, c) for c in caps]
            steps = iter(self.autoregressive.generate_grouped_stream(
                autos, toks, caps, first, block, uniforms_list=us, pos_mode=self._pos_mode(), use_graph=timed, **dec))
            while True:
                e0, e1 = new_event(), new_event()
                record(e0)
                try:
                    codes, ended, lat = next(steps)
                except StopIteration:
                    break
                record(e1)
                ar_parts.append((e0, e1))
                jobs = {}                                  # token count -> [(row, flushes)]
                for u in range(R):
                    if done[u]:
                        continue
                    n = int(codes[u].numel())
                    flags = stream_flushes(n, flushed[u], ended[u], flush_every)
                    if flags:
                        jobs.setdefault(n, []).append((u, flags))
                    if ended[u]:
                        done[u], tokens[u] = True, n
                for n in sorted(jobs):
                    rows = [u for u, _ in jobs[n]]
                    h0, h1 = new_event(), new_event()
                    record(h0)
                    wavs = self.hifi_decoder.inference_batch(lat[rows, :n], torch.stack([autos[u] for u in rows]))
                    record(h1)
                    hifi_parts.append((h0, h1))
                    for (u, flags), wav_gen in zip(jobs[n], wavs):
                        for i, is_end in enumerate(flags):
                            # tts_stream decodes every flush into a buffer of its own, and handle_chunks fades in place
                            w = wav_gen if i == 0 else wav_gen.clone()
                            chunk, wav_prev[u], wav_tail[u] = self.handle_chunks(w, wav_prev[u], wav_tail[u],
                                                                                 overlap_wav_len)
                            flushed[u] = n
                            yield u, chunk, is_end
            end = new_event()
            record(end)
        self.last_timings = {"tokens": tokens}
        if timed:
            end.synchronize()
            self.last_timings = {"ar_ms": sum(a.elapsed_time(b) for a, b in ar_parts),
                                 "hifigan_ms": sum(a.elapsed_time(b) for a, b in hifi_parts),
                                 "device_total_ms": start.elapsed_time(end), "tokens": tokens}

    def stream_pool(self, max_streams=64, overlap_wav_len=1024, stream_chunk_size=40, temperature=.8, length_penalty=1,
                    repetition_penalty=2.0, top_p=.8, max_mel_tokens=500, cvvp_amount=.0, diffusion_iterations=100,
                    cond_free=True, cond_free_k=2, diffusion_temperature=1.0, top_k=50, k=1, verbose=True,
                    num_autoregressive_samples=512, return_deterministic_state=False, **hf_generate_kwargs):
        """A StreamPool of `max_streams` (1..256) slots: texts submitted at any time stream from one running decode
        batch. The keyword arguments are tts_stream's, accepted and rejected as it does; they are every stream's
        defaults, which StreamPool.submit may override per stream."""
        if hf_generate_kwargs:
            raise TypeError(f"unsupported generate kwargs: {sorted(hf_generate_kwargs)}")
        if not 1 <= int(max_streams) <= lib.AR_STEP_MAX_GROUPS:
            raise ValueError("max_streams must lie in 1..%d, got %r" % (lib.AR_STEP_MAX_GROUPS, max_streams))
        dec = dict(temperature=temperature, top_k=top_k, top_p=top_p, repetition_penalty=repetition_penalty)
        return StreamPool(self, int(max_streams), overlap_wav_len, int(stream_chunk_size), dec)

    def tts_long_stream(self, text, voice_samples=None, text_tokens_list=None, **kwargs):
        """≙ the loop of the reference's `tts_stream.py` for one voice: split the text (`'|'` forces the split points,
        else `split_and_recombine_text`) and stream every chunk with the SAME seed, as 1-D waveform chunks in playback
        order: all of sentence 0, then sentence 1, and so on. The sentences are streamed by tts_stream_batch, up to 256
        per batch (consecutive batches beyond that), so later sentences decode while the first ones play; a sentence
        whose prompt is longer than 352 positions is streamed alone by tts_stream. `text_tokens_list` (one id list per
        chunk) bypasses the tokenizer; the other keyword arguments are those of tts_stream."""
        from .ar_engine import plan_batches
        from .text import split_and_recombine_text
        texts = text.split("|") if "|" in text else split_and_recombine_text(text)
        if text_tokens_list is not None and len(text_tokens_list) != len(texts):
            raise ValueError("text_tokens_list has %d entries for %d chunks" % (len(text_tokens_list), len(texts)))
        raw = [[int(t) for t in (text_tokens_list[u] if text_tokens_list is not None else self.tokenizer.encode(texts[u]))]
               for u in range(len(texts))]
        return self._long_stream(texts, raw, voice_samples, kwargs,
                                 plan_batches([(1, len(t) + 5) for t in raw], max_groups=lib.AR_STEP_MAX_GROUPS))

    def _long_stream(self, texts, raw, voice_samples, kwargs, batches):
        kwargs = dict(kwargs)
        kwargs["use_deterministic_seed"] = self.deterministic_state(seed=kwargs.get("use_deterministic_seed"))
        for batch in batches:
            if len(batch) == 1 and len(raw[batch[0]]) + 5 > lib.AR_STEP_MAX_P:
                yield from self.tts_stream(texts[batch[0]], voice_samples=voice_samples, text_tokens=raw[batch[0]],
                                           **kwargs)
                continue
            pending = [[] for _ in batch]              # chunks of sentences after the one playing
            finished = [False] * len(batch)
            cur = 0
            for u, chunk, last in self.tts_stream_batch([texts[i] for i in batch], voice_samples=voice_samples,
                                                        text_tokens_list=[raw[i] for i in batch], **kwargs):
                if u == cur:
                    yield chunk
                else:
                    pending[u].append(chunk)
                finished[u] = finished[u] or last
                while cur < len(batch) and finished[cur]:
                    cur += 1
                    if cur < len(batch):
                        yield from pending[cur]
                        pending[cur] = []


def _whole(name, v):
    """v as an int; ValueError unless it is a whole number."""
    try:
        i = int(v)
    except (TypeError, ValueError):
        raise ValueError("%s must be an integer, got %r" % (name, v)) from None
    if isinstance(v, bool) or i != v:
        raise ValueError("%s must be an integer, got %r" % (name, v))
    return i


class StreamPool:
    """Continuous batching of tts_stream: texts join a decode batch that is already running, each in a free slot, and
    leave it when they end. The chunks of stream `sid` are those of `tts_stream(text, voice_samples=...,
    text_tokens=..., use_deterministic_seed=seed, **the pool's kwargs)`: the same tokens, chunk count and lengths,
    `last` on the final chunk, whenever the text was submitted and whatever else runs. The latents come from the decode
    steps (as in tts_stream_batch), so the samples agree with tts_stream's within rounding (DESIGN §5).

    Each stream has its own voice and seed: its uniforms row and its conditioning crop follow the seed as in tts_stream.
    Each stream may also have its own sampling settings, chunk size and cross-fade (`submit`); the pool's kwargs are
    the defaults. The settings sit in a per-row table on the device. While every stream has the pool's settings the
    decode samples with the scalar sampler, as before; the first stream with settings of its own switches the pool to
    the per-row sampler (ttb_ar_sample_params), whose step graph is captured once, then. A full pool queues texts first in,
    first out; the pool looks at its queue at least every POOL_ADMIT_STEPS (16) decode steps, so a text starts decoding
    within 16 steps of a slot being free. `submit` may be called from any thread; every CUDA call happens on the thread
    that iterates the pool (`poll` / `run`). Every stream applies stream_flushes to its own token count and ends at its
    stop token (found no later than its next flush point) or at its cap of 500 - P tokens; its slot is then refilled
    from the queue. HiFiGAN decodes the rows that flush at the same token count in one inference_batch pass.

    `last_timings[sid]` (set when stream sid ends): tokens, wait_admit_s (submit to admission) and wait_first_chunk_s
    (submit to first chunk, host clock); on the GPU also ar_ms (device time of the decode steps while it ran), prefill_ms
    (its admission prefill) and hifigan_ms (the HiFiGAN passes it took part in)."""

    def __init__(self, tts, max_streams, overlap_wav_len, flush_every, dec):
        self.tts, self.capacity = tts, max_streams
        self.overlap, self.flush_every, self.dec = overlap_wav_len, flush_every, dec
        self.timed = tts.device.type == "cuda"
        self.ws = tts.autoregressive.slot_workspace(max_streams, STREAM_MAX_LENGTH, pos_mode=tts._pos_mode(),
                                                    use_graph=self.timed, **dec)
        self.slots = [None] * max_streams
        self.last_timings = {}
        self._lock = threading.Lock()
        self._queue = collections.deque()
        self._next_sid = 0
        self._closed = False
        self._ar_pending = []                          # (start, end, streams running) of decode steps not yet read

    def submit(self, text, voice_samples=None, conditioning_latent=None, text_tokens=None, use_deterministic_seed=None,
               temperature=None, top_p=None, top_k=None, repetition_penalty=None, length_penalty=None,
               stream_chunk_size=None, overlap_wav_len=None):
        """Queues a text; returns its stream id. `conditioning_latent` (an auto latent as get_conditioning_latents
        returns it) excludes `voice_samples`; neither = a random voice, as in tts_stream. A prompt longer than 352
        positions raises ValueError (tts_stream can stream it alone).
        temperature, top_p, top_k, repetition_penalty, stream_chunk_size and overlap_wav_len: this stream's own, as
        tts_stream takes them; None = the pool's. length_penalty is accepted and has no effect, as in tts_stream. The
        stream's chunks are then those of tts_stream(text, ..., **{**the pool's kwargs, **these}). A bad value raises
        ValueError here, before anything is queued."""
        if voice_samples is not None and conditioning_latent is not None:
            raise ValueError("give voice_samples or conditioning_latent, not both")
        given = dict(temperature=temperature, top_p=top_p, top_k=top_k, repetition_penalty=repetition_penalty)
        settings = {k: v for k, v in given.items() if v is not None}
        lib.sample_params_row(**{**self.dec, **settings})
        every = self.flush_every if stream_chunk_size is None else _whole("stream_chunk_size", stream_chunk_size)
        overlap = self.overlap if overlap_wav_len is None else _whole("overlap_wav_len", overlap_wav_len)
        toks = self.tts._inputs_tokens(text, text_tokens)
        if len(toks) + 4 > lib.AR_STEP_MAX_P:
            raise ValueError("a prompt of %d positions (a pool slot holds %d; tts_stream streams it alone)" %
                             (len(toks) + 4, lib.AR_STEP_MAX_P))
        with self._lock:
            if self._closed:
                raise RuntimeError("the stream pool is closed")
            sid = self._next_sid
            self._next_sid += 1
            self._queue.append(dict(sid=sid, toks=toks, voice=voice_samples, cond=conditioning_latent,
                                    seed=use_deterministic_seed, settings=settings, every=every, overlap=overlap,
                                    t_submit=perf_counter()))
        return sid

    def _event(self):
        if not self.timed:
            return None
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        return e

    def _fill(self):
        """Admits queued texts into free slots, first in, first out."""
        for slot in range(self.capacity):
            if self.slots[slot] is not None:
                continue
            with self._lock:
                if not self._queue:
                    return
                rec = self._queue.popleft()
            self._admit(slot, rec)

    def _admit(self, slot, rec):
        tts = self.tts
        seed = tts.deterministic_state(seed=rec["seed"])
        auto = rec["cond"].to(tts.device).float().reshape(-1) if rec["cond"] is not None else \
            tts._auto_latent(rec["voice"])
        P = len(rec["toks"]) + 4
        cap = STREAM_MAX_LENGTH - P
        every = rec["every"]
        first = max(every, FIRST_BUFFER) if every > 0 else cap
        e0 = self._event()
        self.ws.admit(slot, auto, rec["toks"], tts._uniforms(seed, cap), rec["settings"])
        e1 = self._event()
        rec.update(auto=auto, cap=cap, block=every if every > 0 else cap, obs=min(first, cap), flushed=0,
                   wav_prev=None, wav_tail=None, t_admit=perf_counter(), t_first=None, prefill=(e0, e1),
                   hifi=[], ar_ms=0.0)
        self.slots[slot] = rec

    def _read_ar(self):
        """Adds the device time of the decode steps recorded so far to the streams they ran (after a synchronise)."""
        for a, b, recs in self._ar_pending:
            ms = a.elapsed_time(b)
            for rec in recs:
                rec["ar_ms"] += ms
        self._ar_pending = []

    def poll(self):
        """Advances the pool to its next event: a list of (sid, chunk, last), or [] when no stream is active or
        queued."""
        stop = self.tts.cfg.stop_mel_token
        ws = self.ws
        while True:
            self._fill()
            active = [s for s in range(self.capacity) if self.slots[s] is not None]
            if not active:
                return []
            n = min(self.slots[s]["obs"] - ws.tokens(s) for s in active)
            n = min(n, POOL_ADMIT_STEPS)
            if n > 0:
                e0 = self._event()
                ws.advance(n)
                if self.timed:
                    self._ar_pending.append((e0, self._event(), [self.slots[s] for s in active]))
            due = [s for s in active if ws.tokens(s) >= self.slots[s]["obs"]]
            if due:
                return self._observe(due, stop)

    def _observe(self, due, stop):
        ws = self.ws
        host = ws.codes().cpu()
        ws.check()
        if self.timed:
            self._read_ar()
        jobs, ended_slots = {}, []
        for s in due:
            rec = self.slots[s]
            h = rec["obs"]
            hit = (host[s, :h] == stop).nonzero()
            if hit.numel() > 0:
                n, ended = int(hit[0].item()) + 1, True
            else:
                n, ended = h, h >= rec["cap"]
            flags = stream_flushes(n, rec["flushed"], ended, rec["every"])
            if flags:
                jobs.setdefault(n, []).append((s, flags))
            if ended:
                rec["tokens"] = n
                ended_slots.append(s)
            else:
                rec["obs"] = min(h + rec["block"], rec["cap"])
        out = []
        lat = ws.latents
        for n in sorted(jobs):
            rows = [s for s, _ in jobs[n]]
            h0 = self._event()
            wavs = self.tts.hifi_decoder.inference_batch(lat[rows, :n], torch.stack([self.slots[s]["auto"] for s in rows]))
            h1 = self._event()
            for (s, flags), wav_gen in zip(jobs[n], wavs):
                rec = self.slots[s]
                rec["hifi"].append((h0, h1))
                for i, is_end in enumerate(flags):
                    # tts_stream decodes every flush into a buffer of its own, and handle_chunks fades in place
                    w = wav_gen if i == 0 else wav_gen.clone()
                    chunk, rec["wav_prev"], rec["wav_tail"] = self.tts.handle_chunks(w, rec["wav_prev"], rec["wav_tail"],
                                                                                      rec["overlap"])
                    rec["flushed"] = n
                    if rec["t_first"] is None:
                        rec["t_first"] = perf_counter()
                    out.append((rec["sid"], chunk, is_end))
        for s in ended_slots:
            self._finish(s)
        return out

    def _finish(self, s):
        rec = self.slots[s]
        self.ws.release(s)
        self.slots[s] = None
        t = {"tokens": rec["tokens"], "wait_admit_s": rec["t_admit"] - rec["t_submit"],
             "wait_first_chunk_s": rec["t_first"] - rec["t_submit"]}
        if self.timed:
            if rec["hifi"]:
                rec["hifi"][-1][1].synchronize()
            t.update(ar_ms=rec["ar_ms"], prefill_ms=rec["prefill"][0].elapsed_time(rec["prefill"][1]),
                     hifigan_ms=sum(a.elapsed_time(b) for a, b in rec["hifi"]))
        self.last_timings[rec["sid"]] = t

    def run(self):
        """Yields (sid, chunk, last) until no stream is active or queued."""
        while True:
            ev = self.poll()
            if not ev:
                return
            yield from ev

    def close(self):
        """Drops the queue and the decode workspace; the pool cannot be used afterwards."""
        with self._lock:
            self._closed = True
            self._queue.clear()
        self.slots = [None] * self.capacity
        self.ws = None
