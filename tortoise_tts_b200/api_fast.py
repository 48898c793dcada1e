"""Drop-in facade for `tortoise.api_fast.TextToSpeech` (tortoise/api_fast.py:171-520) on the sm_90a engine: the
reference's low-latency product path — ONE autoregressive sequence, no CLVP / diffusion, GPT latents rendered
directly by the HiFiGAN decoder (`hifidecoder.pth`), optionally streamed chunk by chunk.

Same constructor, `tts()`, `tts_stream()`, `tts_with_preset()`, `handle_chunks()`, `get_conditioning_latents()`
(auto latent only, api_fast.py:225-246), `get_random_conditioning_latents()` (api_fast.py:248-254) and
`deterministic_state()`. Everything between the tokenizer and the returned waveform runs in libttb.so: the decode
loop (`AREngine.generate` / `generate_stream`), the latent pass (`AREngine.latents` / `stream_latents`) and the
decoder (`HifiganEngine`).

Deliberate differences (SURVEY App. D): sampling randomness comes from a device generator seeded by
`use_deterministic_seed`; `tts_with_preset` drops the diffusion-only preset keys instead of forwarding them to HF
`generate` (which rejects them in the reference); the wav2vec redaction model is not loaded.
"""
import os
import random
from time import time

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
        if text_tokens is None:
            text_tokens = self.tokenizer.encode(text)
        toks = [int(t) for t in text_tokens] + [0]            # F.pad(text_tokens, (0, 1))
        assert len(toks) < 400, "Too much text provided. Break the text up into separate segments and re-try inference."
        if voice_samples is not None:
            auto = self.get_conditioning_latents(voice_samples, return_mels=False)
        else:
            auto = self.get_random_conditioning_latents()
        return seed, toks, auto.to(self.device).float().reshape(-1)

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
                # the reference flushes when the tokens buffered since the last flush reach the threshold, and once more
                # when the generator is exhausted (even if nothing new arrived since the last flush)
                due = flush_every > 0 and (n - flushed) >= (first if flushed == 0 else flush_every)
                for is_end in ([False] if due else []) + ([True] if ended else []):
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
            g = torch.Generator(device=self.device)
            g.manual_seed(seed)
            uniforms = torch.rand(1, n_max, generator=g, device=self.device)
            codes = self.autoregressive.generate(auto, toks, 1, n_max, uniforms=uniforms, temperature=temperature,
                                                 top_k=top_k, top_p=top_p, repetition_penalty=repetition_penalty,
                                                 pos_mode=self._pos_mode(), use_graph=self.device.type == "cuda",
                                                 typical_mass=typical)
            hit = (codes[0] == self.cfg.stop_mel_token).nonzero()
            n = int(hit[0].item()) + 1 if hit.numel() > 0 else n_max          # HF returns the stop token it sampled
            mark(1)
            if verbose:
                print("generating audio..")
            lat = self.autoregressive.latents(auto, toks, codes[:, :n].contiguous())[0]
            mark(2)
            wav = self.hifi_decoder.inference(lat, auto)
            mark(3)
        self.last_timings = {"tokens": n}
        if timed:
            torch.cuda.synchronize()
            self.last_timings = {"ar_ms": ev[0].elapsed_time(ev[1]), "latents_ms": ev[1].elapsed_time(ev[2]),
                             "hifigan_ms": ev[2].elapsed_time(ev[3]), "tokens": n}
        return wav.reshape(1, 1, -1)
