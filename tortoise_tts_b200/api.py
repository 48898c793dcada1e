"""Drop-in facade for `tortoise.api.TextToSpeech` (tortoise/api.py:174-609) on the sm_90a engine.

Same constructor / `tts()` / `tts_with_preset()` signatures, presets, return types and checkpoint layout
(`models_dir` with autoregressive.pth, diffusion_decoder.pth, clvp2.pth, vocoder.pth). Everything between the
tokenizer and `wav.cpu()` runs in libttb.so; there is no PyTorch/CPU fallback for the hot path.

Differences that are deliberate (SURVEY App. D): all candidates are decoded in one batch (the reference loops over
`autoregressive_batch_size` chunks and silently drops the remainder), models stay resident on the device, and the
sampling / diffusion randomness comes from device generators seeded by `use_deterministic_seed`.
"""
import os
import random
from time import time, perf_counter

import torch

from .config import ModelConfig
from .ar_engine import AREngine
from .clvp_engine import CLVPEngine
from .diffusion_engine import DiffusionEngine
from .vocoder_engine import VocoderEngine
from .conditioning_engine import ConditioningEngine, RandomLatentEngine
from . import lib
from . import parallel

DEFAULT_MODELS_DIR = os.path.join(os.path.expanduser("~"), ".cache", "tortoise", "models")
MODELS_DIR = os.environ.get("TORTOISE_MODELS_DIR", DEFAULT_MODELS_DIR)
# the two Hugging Face repositories Wav2VecAlignment loads (utils/wav2vec_alignment.py:53,55)
ALIGNER_REPOS = ("jbetker/wav2vec2-large-robust-ft-libritts-voxpopuli", "jbetker/tacotron-symbols")
MODELS = ("autoregressive.pth", "classifier.pth", "clvp2.pth", "cvvp.pth", "diffusion_decoder.pth", "vocoder.pth",
          "rlg_auto.pth", "rlg_diffuser.pth")

PRESETS = {  # api.py:320-329
    "ultra_fast": {"num_autoregressive_samples": 16, "diffusion_iterations": 30, "cond_free": False},
    "fast": {"num_autoregressive_samples": 96, "diffusion_iterations": 80},
    "standard": {"num_autoregressive_samples": 256, "diffusion_iterations": 200},
    "high_quality": {"num_autoregressive_samples": 256, "diffusion_iterations": 400},
}


def get_model_path(model_name, models_dir=MODELS_DIR):
    if model_name not in MODELS:
        raise ValueError(f"Model {model_name} not found in available models.")
    path = os.path.join(models_dir, model_name)
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path} missing (this build is offline: place the reference checkpoints there)")
    return path


def pad_or_truncate(t, length):
    if t.shape[-1] == length:
        return t
    if t.shape[-1] < length:
        return torch.nn.functional.pad(t, (0, length - t.shape[-1]))
    return t[..., :length]


def _default_mel_norms():
    """tortoise/data/mel_norms.pth (TorchMelSpectrogram's per-bin divisors): TORTOISE_MEL_NORMS (.pth) overrides the
    packaged copy of the 80 numbers."""
    p = os.environ.get("TORTOISE_MEL_NORMS")
    if p:
        return torch.load(p, map_location="cpu").float()
    import json
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "data", "mel_norms.json")) as f:
        return torch.tensor(json.load(f)["mel_norms"], dtype=torch.float32)


class DiffuserSpec:
    """What `load_discrete_vocoder_diffuser` (api.py:64-70) configures: the number of respaced steps of the 4000-step
    linear schedule and the classifier-free-guidance setting. The schedule tables themselves live on the device inside
    DiffusionEngine (same float64 construction as SpacedDiffusion, diffusion_engine.make_schedule)."""

    def __init__(self, trained_diffusion_steps=4000, desired_diffusion_steps=200, cond_free=True, cond_free_k=1):
        if trained_diffusion_steps != 4000:
            raise ValueError("the engine's schedule is the reference's 4000-step linear schedule")
        self.num_timesteps = int(desired_diffusion_steps)
        self.conditioning_free = bool(cond_free)
        self.conditioning_free_k = float(cond_free_k)


def load_discrete_vocoder_diffuser(trained_diffusion_steps=4000, desired_diffusion_steps=200, cond_free=True, cond_free_k=1):
    """≙ api.py:64-70."""
    return DiffuserSpec(trained_diffusion_steps, desired_diffusion_steps, cond_free, cond_free_k)


def format_conditioning(clip, cond_length=132300, device="cuda", engine=None):
    """≙ api.py:73-84: clip [1, n] at 22.05 kHz -> MEL [1, 80, 517] (random crop via `random`, as the reference).
    `engine`: a ConditioningEngine (TextToSpeech.conditioning); built on demand from the packaged mel_norms otherwise."""
    if cond_length != 132300:
        raise ValueError("cond_length is fixed at 132300 samples (the ConditioningEncoder's training length)")
    if engine is None:
        engine = _MelOnly(device)
    w = ConditioningEngine.format_clip(clip.to(engine.dev).float()).contiguous()
    mf = torch.empty(80, 1 + w.numel() // 256, dtype=torch.float32, device=engine.dev)
    engine.ar_mel(w, mf)
    return mf.unsqueeze(0)


class _MelOnly(ConditioningEngine):
    """The table part of ConditioningEngine (no encoder weights): enough for format_conditioning()."""

    def __init__(self, device):
        import numpy as np
        from .conditioning_engine import _mel_filterbank, N_FFT
        self.dev = torch.device(device)
        n = np.arange(N_FFT)
        self.window = torch.from_numpy(0.5 - 0.5 * np.cos(2.0 * np.pi * n / N_FFT)).float().to(self.dev)
        tw = np.stack([np.cos(2.0 * np.pi * n / N_FFT), np.sin(2.0 * np.pi * n / N_FFT)], axis=1)
        self.twiddle = torch.from_numpy(tw).float().contiguous().to(self.dev)
        self.fb_ar = torch.from_numpy(_mel_filterbank(22050, N_FFT, 80, 0.0, 8000.0, "htk")).float().contiguous().to(self.dev)
        self.mel_norms = _default_mel_norms().to(self.dev)
        self.kpad_ar = 128


def fix_autoregressive_output(codes, stop_token, complain=True):
    """≙ api.py:87-114 on one row of codes (1-D integer tensor): in place on the device, returns the tensor."""
    if codes.dim() != 1:
        raise ValueError("fix_autoregressive_output works on one row of codes (api.py:87-114)")
    work = codes.to(device="cuda", dtype=torch.int32).contiguous()
    has_stop = bool((work == stop_token).any().item())
    if not has_stop:
        if complain:
            print("No stop tokens found in one of the generated voice clips. This typically means the spoken audio is "
                  "too long. In some cases, the output will still be good, though. Listen to it and if it is missing words, "
                  "try breaking up your input text.")
        return codes
    lib.ar_fix_codes(work, 1, work.numel(), int(stop_token), None)
    codes.copy_(work.to(device=codes.device, dtype=codes.dtype))
    return codes


def do_spectrogram_diffusion(diffusion_model, diffuser, latents, conditioning_latents, temperature=1, verbose=True):
    """≙ api.py:117-130. diffusion_model: DiffusionEngine (TextToSpeech.diffusion); diffuser: DiffuserSpec; latents
    [1, N, D]; conditioning_latents [1, 2C]. Noise comes from torch's generator of the model's device, as in the reference.
    Returns the denormalised MEL [1, 100, S]."""
    if latents.shape[0] != 1:
        raise ValueError("the reference's diffusion sampler is batch-1 (utils/diffusion.py:379)")
    dev = diffusion_model.dev
    lat = latents[0].to(dev).float().contiguous()
    S = lat.shape[0] * 4 * 24000 // 22050
    iters = diffuser.num_timesteps
    noise0 = torch.randn(100, S, device=dev) * temperature
    step_noise = torch.randn(iters, 100, S, device=dev)
    mel = diffusion_model.sample(lat, conditioning_latents.to(dev).float().reshape(-1), iters, noise0, step_noise,
                                 cond_free=diffuser.conditioning_free, cond_free_k=diffuser.conditioning_free_k)
    return mel.unsqueeze(0)


def _typical_mass(typical_sampling, typical_mass):
    """The engine's typical_mass for the tts() kwargs `typical_sampling` / `typical_mass`: None when the filter is off.
    A mass outside (0, 1] raises ValueError. The reference raises an IndexError where the cumulative mass never reaches
    typical_mass (mass 1 under rounding); here every token is kept instead."""
    if not typical_sampling:
        return None
    m = float(typical_mass)
    if not 0.0 < m <= 1.0:
        raise ValueError("typical_mass must lie in (0, 1], got %r" % (typical_mass,))
    return m


_CLASSIFIERS = {}


def classify_audio_clip(clip, models_dir=MODELS_DIR):
    """≙ api.py:133-145: the probability that the tortoise-detect classifier (AudioMiniEncoderWithClassifierHead)
    assigns to class 0 of `clip`, a [1, n] float waveform at 24 kHz on any device, as a 0-d float32 CPU tensor
    (softmax(logits)[0][0]). Any other shape raises ValueError.

    Deliberate differences: the classifier runs on the current CUDA device (classifier_engine.py), not on the CPU; and
    `classifier.pth` is loaded on the first call and the packed engine is kept per (checkpoint path, device), where the
    reference reloads the checkpoint on every call."""
    if not torch.is_tensor(clip) or clip.dim() != 2 or clip.shape[0] != 1 or clip.shape[1] < 1 \
            or not clip.is_floating_point():
        raise ValueError("classify_audio_clip expects a float waveform of shape [1, n], got %s" %
                         ((tuple(clip.shape) if torch.is_tensor(clip) else type(clip).__name__),))
    from .classifier_engine import ClassifierEngine
    path = os.path.abspath(get_model_path("classifier.pth", models_dir))
    dev = torch.device("cuda", torch.cuda.current_device())
    eng = _CLASSIFIERS.get((path, dev))
    if eng is None:
        eng = _CLASSIFIERS[(path, dev)] = ClassifierEngine(torch.load(path, map_location="cpu", weights_only=True), dev)
    _, probs = eng.forward(clip)
    return probs[0, 0].cpu()


def pick_best_batch_size_for_gpu():
    """≙ api.py:148-172 (kept for callers; this engine decodes all candidates in one batch regardless)."""
    if torch.cuda.is_available():
        _, available = torch.cuda.mem_get_info()
        gb = available / (1024 ** 3)
        if gb > 14:
            return 16
        if gb > 10:
            return 8
        if gb > 7:
            return 4
    return 1


class _Tokenizer:
    """VoiceBpeTokenizer (utils/tokenizer.py:172-197): `english_cleaners` by default, `basic_cleaners` with
    `use_basic_cleaners` (the constructor's `tokenizer_basic`). The BPE vocabulary is the reference's data/tokenizer.json
    (an asset, not code): pass `tokenizer_vocab_file` or set TORTOISE_TOKENIZER_JSON."""

    def __init__(self, vocab_file=None, use_basic_cleaners=False):
        from tokenizers import Tokenizer
        from . import cleaners
        self.preprocess_text = cleaners.basic_cleaners if use_basic_cleaners else cleaners.english_cleaners
        vocab_file = vocab_file or os.environ.get("TORTOISE_TOKENIZER_JSON")
        if vocab_file is None or not os.path.exists(vocab_file):
            raise FileNotFoundError("tokenizer.json not found: pass tokenizer_vocab_file=... (reference asset "
                                    "tortoise/data/tokenizer.json) or call tts() with pre-tokenised `text_tokens`")
        self.tok = Tokenizer.from_file(vocab_file)

    def encode(self, txt):
        txt = self.preprocess_text(txt)
        txt = txt.replace(" ", "[SPACE]")
        return self.tok.encode(txt).ids

    def decode(self, seq):
        if isinstance(seq, torch.Tensor):
            seq = seq.cpu().numpy()
        txt = self.tok.decode(seq, skip_special_tokens=False).replace(" ", "")
        return txt.replace("[SPACE]", " ").replace("[STOP]", "").replace("[UNK]", "")


def _hf_cache_snapshot(repo):
    """Directory of the cached snapshot of a Hugging Face repository, found on disk only (no network), or None."""
    home = os.environ.get("HF_HOME", os.path.join(os.path.expanduser("~"), ".cache", "huggingface"))
    for root in (os.environ.get("HF_HUB_CACHE"), os.path.join(home, "hub")):
        if not root:
            continue
        d = os.path.join(root, "models--" + repo.replace("/", "--"))
        ref = os.path.join(d, "refs", "main")
        if os.path.exists(ref):
            with open(ref) as f:
                snap = os.path.join(d, "snapshots", f.read().strip())
            if os.path.isdir(snap):
                return snap
        snaps = os.path.join(d, "snapshots")
        if os.path.isdir(snaps) and os.listdir(snaps):
            return os.path.join(snaps, sorted(os.listdir(snaps))[-1])
    return None


class TextToSpeech:
    def __init__(self, autoregressive_batch_size=None, models_dir=MODELS_DIR, enable_redaction=True, kv_cache=False,
                 use_deepspeed=False, half=False, device=None, tokenizer_vocab_file=None, tokenizer_basic=False,
                 state_dicts=None, config: ModelConfig = None, aligner_dir=None):
        """`state_dicts` (dict with keys autoregressive/diffusion/clvp/vocoder) bypasses models_dir (synthetic
        checkpoints); `config` overrides the full-size ModelConfig (tests).

        With `enable_redaction` (the default, as in the reference) the `[bracketed]` parts of a text are cut from the
        returned audio by a wav2vec2 CTC aligner, loaded at the first such text from: state_dicts["wav2vec"] =
        (config, state dict, vocab) (synth.synth_wav2vec), else `aligner_dir` / TORTOISE_WAV2VEC_DIR (an HF checkpoint
        directory; vocab.json from TORTOISE_WAV2VEC_VOCAB or that directory), else the local Hugging Face cache of
        ALIGNER_REPOS."""
        if not torch.cuda.is_available():
            raise RuntimeError("tortoise_tts_b200 needs a CUDA device (sm_90a); there is no CPU path")
        lib.load()
        self.models_dir = models_dir
        self.autoregressive_batch_size = autoregressive_batch_size  # accepted for API parity; one batch is used
        self.enable_redaction = bool(enable_redaction)
        self._aligner_dir = aligner_dir
        self.aligner = None              # loaded at the first tts() text with a '[' (load_aligner)
        self.kv_cache = kv_cache
        self.device = torch.device(device if device is not None else "cuda")
        if self.device.type == "cuda":
            # the kernels are enqueued on the CURRENT device's stream: make the engine's device current (weights,
            # workspaces and launches must agree; reference api.py:202-205 only records the device)
            torch.cuda.set_device(self.device if self.device.index is not None else torch.cuda.current_device())
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.cfg = config or ModelConfig.full()
        self._tok_file = tokenizer_vocab_file
        self._tok_basic = bool(tokenizer_basic)
        self._tokenizer = None
        if state_dicts is None:
            state_dicts = {
                "autoregressive": torch.load(get_model_path("autoregressive.pth", models_dir), map_location="cpu"),
                "diffusion": torch.load(get_model_path("diffusion_decoder.pth", models_dir), map_location="cpu"),
                "clvp": torch.load(get_model_path("clvp2.pth", models_dir), map_location="cpu"),
                "vocoder": torch.load(get_model_path("vocoder.pth", models_dir), map_location="cpu")["model_g"],
            }
        self.autoregressive = AREngine(state_dicts["autoregressive"], self.cfg, self.device)
        self.clvp = CLVPEngine(state_dicts["clvp"], self.cfg, self.device)
        self.diffusion = DiffusionEngine(state_dicts["diffusion"], self.cfg, self.device)
        self.vocoder = VocoderEngine(state_dicts["vocoder"], self.cfg, self.device)
        self.conditioning = ConditioningEngine(state_dicts["autoregressive"], state_dicts["diffusion"], self.cfg,
                                               self.device, mel_norms=state_dicts.get("mel_norms", None)
                                               if state_dicts.get("mel_norms", None) is not None else _default_mel_norms())
        self._rlg_sd = (state_dicts.get("rlg_auto"), state_dicts.get("rlg_diffuser"))
        self.rlg_auto = self.rlg_diffusion = None
        self._cvvp_sd = state_dicts.get("cvvp")
        self._wav2vec = state_dicts.get("wav2vec")
        self.cvvp = None                 # the CVVP model is only loaded if used (api.py:234,252-256)
        self.last_timings = {}
        self.debug_capture = False
        self.last_debug = None

    def get_conditioning_latents(self, voice_samples, return_mels=False):
        """≙ api.py:258-299: list of reference clips (22.05 kHz waveforms [1, n]) -> (auto latent [1, D], diffusion latent
        [1, 2C]) [+ the two stacks of conditioning MELs]."""
        if not isinstance(voice_samples, (list, tuple)):
            voice_samples = [voice_samples]
        with torch.no_grad():
            if return_mels:
                auto_latent, auto_conds = self.conditioning.ar_latent(voice_samples, return_mels=True)
                diffusion_latent, diffusion_conds = self.conditioning.diffusion_latent(voice_samples, return_mels=True)
                return auto_latent, diffusion_latent, auto_conds, diffusion_conds
            return self.conditioning.ar_latent(voice_samples), self.conditioning.diffusion_latent(voice_samples)

    def load_cvvp(self):
        """≙ api.py:252-256 (cvvp.pth, lazily loaded)."""
        from .cvvp_engine import CVVPEngine
        sd = self._cvvp_sd
        if sd is None:
            sd = torch.load(get_model_path("cvvp.pth", self.models_dir), map_location="cpu")
        self.cvvp = CVVPEngine(sd, self.cfg, self.device)

    def load_aligner(self):
        """The wav2vec2 aligner of prompt redaction (Wav2VecAlignment, api.py:204-205); see __init__ for the sources."""
        from .redaction import Aligner, CTCCharTokenizer
        from .wav2vec_engine import Wav2VecEngine, load_checkpoint
        if self._wav2vec is not None:
            cfg, sd, vocab = self._wav2vec
            tok = CTCCharTokenizer(vocab)
        else:
            mdir = self._aligner_dir or os.environ.get("TORTOISE_WAV2VEC_DIR")
            vocab = os.environ.get("TORTOISE_WAV2VEC_VOCAB")
            if vocab is None and mdir and os.path.exists(os.path.join(mdir, "vocab.json")):
                vocab = mdir
            mdir = mdir or _hf_cache_snapshot(ALIGNER_REPOS[0])
            vocab = vocab or _hf_cache_snapshot(ALIGNER_REPOS[1])
            if not mdir or not os.path.exists(os.path.join(mdir, "config.json")) or not vocab:
                raise FileNotFoundError(
                    "prompt redaction needs the wav2vec2 aligner: pass aligner_dir=... or set TORTOISE_WAV2VEC_DIR (and "
                    "TORTOISE_WAV2VEC_VOCAB), or place %s and %s in the local Hugging Face cache; or construct "
                    "TextToSpeech(enable_redaction=False)" % ALIGNER_REPOS)
            cfg, sd = load_checkpoint(mdir)
            tok = CTCCharTokenizer.from_path(vocab)
        self.aligner = Aligner(Wav2VecEngine(cfg, sd, self.device), tok)

    def get_random_conditioning_latents(self):
        """≙ api.py:301-309 (rlg_auto.pth / rlg_diffuser.pth, lazily loaded)."""
        if self.rlg_auto is None:
            sa, sd_ = self._rlg_sd
            if sa is None:
                sa = torch.load(get_model_path("rlg_auto.pth", self.models_dir), map_location="cpu")
                sd_ = torch.load(get_model_path("rlg_diffuser.pth", self.models_dir), map_location="cpu")
            self.rlg_auto = RandomLatentEngine(sa, self.cfg.ar_dim, self.device)
            self.rlg_diffusion = RandomLatentEngine(sd_, 2 * self.cfg.diff_dim, self.device)
        with torch.no_grad():
            return self.rlg_auto(), self.rlg_diffusion()

    @property
    def tokenizer(self):
        if self._tokenizer is None:
            self._tokenizer = _Tokenizer(self._tok_file, self._tok_basic)
        return self._tokenizer

    def deterministic_state(self, seed=None):
        if seed is None:
            seed = int(time())
            # every rank must derive the SAME candidates table / diffusion noise (the CFG pair mixes branches computed on
            # two ranks against each rank's local x): rank 0's clock decides
            seed = parallel.broadcast_seed(seed, self.device)
        torch.manual_seed(seed)
        random.seed(seed)
        return seed

    def tts_with_preset(self, text, preset="fast", **kwargs):
        settings = {"temperature": .8, "length_penalty": 1.0, "repetition_penalty": 2.0, "top_p": .8,
                    "cond_free_k": 2.0, "diffusion_temperature": 1.0}
        settings.update(PRESETS[preset])
        settings.update(kwargs)
        return self.tts(text, **settings)

    def tts_long(self, text, preset="standard", shard_utterances=True, text_tokens_list=None, **kwargs):
        """≙ the loop of the reference's `read.py:44-85` for one voice: split the text (`'|'` forces the split points,
        else `split_and_recombine_text`), synthesise every chunk with the SAME seed and conditioning latents, and
        concatenate the waveforms (k = 1). Returns `[1, samples]` on the CPU.

        With several ranks and `shard_utterances`, chunk u is rendered WHOLE by rank u % G (SURVEY §8e config 5: no
        collective inside an utterance, so the per-step latency floor of the candidate-sharded mode does not apply)
        and the waveforms are exchanged once at the end. `text_tokens_list` (one id list per chunk) bypasses the
        tokenizer, as `text_tokens` does for `tts()`."""
        from .text import split_and_recombine_text, utterance_plan
        if kwargs.get("k", 1) != 1:
            raise NotImplementedError("tts_long concatenates one waveform per chunk (read.py:77-79): k must be 1")
        texts = text.split("|") if "|" in text else split_and_recombine_text(text)      # read.py:46-52
        if text_tokens_list is not None and len(text_tokens_list) != len(texts):
            raise ValueError("text_tokens_list has %d entries for %d chunks" % (len(text_tokens_list), len(texts)))
        rank, ws = parallel.world()
        spread = bool(shard_utterances) and ws > 1
        plan = utterance_plan(len(texts), ws if spread else 1)
        parts = {}
        for u, chunk in enumerate(texts):
            kw = dict(kwargs)
            if text_tokens_list is not None:
                kw["text_tokens"] = text_tokens_list[u]
            if spread:
                if plan[u] != rank:
                    continue
                with parallel.single_rank():
                    parts[u] = self.tts_with_preset(chunk, preset=preset, **kw).reshape(-1)
            else:
                parts[u] = self.tts_with_preset(chunk, preset=preset, **kw).reshape(-1)
        if spread:
            wavs = parallel.exchange_utterances(parts, plan, self.device)
        else:
            wavs = [parts[u] for u in range(len(texts))]
        return torch.cat([w.reshape(1, -1).cpu() for w in wavs], dim=-1)

    def tts(self, text, voice_samples=None, conditioning_latents=None, k=1, verbose=True, use_deterministic_seed=None,
            return_deterministic_state=False, num_autoregressive_samples=512, temperature=.8, length_penalty=1,
            repetition_penalty=2.0, top_p=.8, max_mel_tokens=500, cvvp_amount=.0, diffusion_iterations=100,
            cond_free=True, cond_free_k=2, diffusion_temperature=1.0, text_tokens=None, top_k=50, typical_sampling=False,
            typical_mass=.9, **hf_generate_kwargs):
        """≙ TextToSpeech.tts (api.py:334-597). `text_tokens` (list of BPE ids) may be given instead of `text`.
        `typical_sampling` / `typical_mass` are the reference's generate kwargs of the same names (api.py:361-364): the
        sampler keeps only the typical set of mass `typical_mass` (in (0, 1]) of the penalised scores."""
        if hf_generate_kwargs:
            raise TypeError(f"unsupported generate kwargs: {sorted(hf_generate_kwargs)}")
        typical = _typical_mass(typical_sampling, typical_mass)
        seed = self.deterministic_state(seed=use_deterministic_seed)
        # api.py:395-401 (after the seeding, so that the random crop / random voice follow use_deterministic_seed)
        auto_conds = None                 # the conditioning MELs: only known when the clips themselves are given
        if voice_samples is not None:
            auto_conditioning, diffusion_conditioning, auto_conds, _ = self.get_conditioning_latents(voice_samples,
                                                                                                   return_mels=True)
            conditioning_latents = (auto_conditioning, diffusion_conditioning)
        elif conditioning_latents is None:
            conditioning_latents = self.get_random_conditioning_latents()
        dev = self.device
        if text_tokens is None:
            text_tokens = self.tokenizer.encode(text)
        toks = [int(t) for t in text_tokens] + [0]            # F.pad(text_tokens, (0, 1)) (api.py:391)
        assert len(toks) < 400, "Too much text provided. Break the text up into separate segments and re-try inference."
        auto_cond, diff_cond = conditioning_latents
        auto_cond = auto_cond.to(dev).float().reshape(-1)
        diff_cond = diff_cond.to(dev).float().reshape(-1)
        rank, ws = parallel.world()
        B = int(num_autoregressive_samples)
        lo, hi = parallel.shard_range(B, rank, ws)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
        with torch.no_grad():
            ev[0].record()
            # sampling randomness is keyed by the GLOBAL candidate id: every rank draws the same [B, N] table and keeps
            # its rows, so results do not depend on the number of GPUs
            g = torch.Generator(device=dev)
            g.manual_seed(seed)
            uniforms = torch.rand(B, max_mel_tokens, generator=g, device=dev)[lo:hi]
            codes = self.autoregressive.generate(auto_cond, toks, hi - lo, max_mel_tokens, uniforms=uniforms,
                                                 temperature=temperature, top_k=top_k, top_p=top_p,
                                                 repetition_penalty=repetition_penalty,
                                                 pos_mode="ref_kv_quirk" if self.kv_cache else "train_consistent",
                                                 typical_mass=typical)
            nb, L = codes.shape
            trim = torch.empty(nb, dtype=torch.int32, device=dev)
            lib.ar_fix_codes(codes, nb, L, self.cfg.stop_mel_token, trim)
            ev[1].record()
            # api.py:450-472: CLVP, CVVP (needs the conditioning mels, i.e. voice_samples) or their blend. cvvp_amount = 1
            # without voice_samples leaves `clvp_out` undefined in the reference; CLVP alone is used here.
            use_cvvp = cvvp_amount > 0 and auto_conds is not None
            if use_cvvp and self.cvvp is None:
                self.load_cvvp()
            scores = None
            if cvvp_amount != 1 or not use_cvvp:
                scores = self.clvp.scores(toks, codes)
            if use_cvvp:
                cv = self.cvvp.scores(auto_conds, codes)
                scores = cv if cvvp_amount == 1 else cv * cvvp_amount + scores * (1 - cvvp_amount)
            scores, codes = parallel.gather_candidates(scores, codes, B)
            best = torch.topk(scores, k=k).indices
            best_codes = codes[best].contiguous()
            if self.debug_capture:      # parity hook (tests): the intermediate results of the stages of this call
                self.last_debug = {"seed": seed, "codes": codes.clone(), "scores": scores.clone(), "best": best.clone(),
                                   "latents": {}, "mel": {}, "noise": {}}
            ev[2].record()
            # rendering plan: candidate j -> owner rank (+ the rank pair sharing its CFG denoiser when ws >= 2)
            use_pair = cond_free and ws >= 2 and os.environ.get("TTB_CFG_PAIR", "1") == "1"   # TTB_CFG_PAIR=0 disables
            groups, _ = parallel.pair_groups() if use_pair else (None, 0)
            plan = [parallel.render_plan(j, ws, use_pair) for j in range(best_codes.shape[0])]
            mine = [j for j, (owner, p) in enumerate(plan) if owner == rank or (p is not None and rank == owner + 1)]
            wavs = {}
            t_lat = t_diff = t_voc = 0.0
            timers = []
            for j in mine:
                e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
                e[0].record()
                lat_full = self.autoregressive.latents(auto_cond, toks, best_codes[j:j + 1])[0]
                e[1].record()
                # calm-token trim (api.py:547-556) on the fixed codes of this candidate
                tl = torch.empty(1, dtype=torch.int32, device=dev)
                lib.ar_fix_codes(best_codes[j:j + 1].clone(), 1, L, self.cfg.stop_mel_token, tl)
                lat = lat_full[: int(tl.item())]
                S = lat.shape[0] * 4 * 24000 // 22050
                gj = torch.Generator(device=dev)
                gj.manual_seed(seed + 7919 * (j + 1))
                noise0 = torch.randn(100, S, generator=gj, device=dev) * diffusion_temperature
                step_noise = torch.randn(diffusion_iterations, 100, S, generator=gj, device=dev)
                owner, p = plan[j]
                pair = None if p is None else (groups[p], rank - owner)
                mel = self.diffusion.sample(lat, diff_cond, diffusion_iterations, noise0, step_noise, cond_free=cond_free,
                                            cond_free_k=cond_free_k, pair=pair)
                e[2].record()
                if self.debug_capture:
                    self.last_debug["latents"][j] = lat.clone()
                    self.last_debug["mel"][j] = mel.clone()
                    self.last_debug["noise"][j] = (noise0.clone(), step_noise.clone())
                if owner == rank:
                    # the reference draws the vocoder noise on the CPU (vocoder.py:307, SURVEY App. D-8); device draw here
                    z = torch.randn(64, S + 10, generator=gj, device=dev)
                    wavs[j] = self.vocoder.inference(mel, z)
                e[3].record()
                timers.append(e)
            ev[3].record()
            t_red = None
            if self.enable_redaction and text is not None and "[" in text:
                # api.py:583-587: every candidate this rank rendered, before the waveforms are exchanged
                if self.aligner is None:
                    self.load_aligner()
                torch.cuda.synchronize()
                t0 = perf_counter()
                for j in wavs:
                    wavs[j] = self.aligner.redact(wavs[j].reshape(1, -1), text)
                torch.cuda.synchronize()
                t_red = (perf_counter() - t0) * 1e3
            res = []
            for j in range(best_codes.shape[0]):
                owner = plan[j][0]
                if ws > 1:
                    n = torch.tensor([wavs[j].numel() if owner == rank else 0], dtype=torch.int64, device=dev)
                    torch.distributed.broadcast(n, src=owner)
                    w = parallel.broadcast_from_owner(wavs.get(j), int(n.item()), owner, dev)
                else:
                    w = wavs[j]
                res.append(w.reshape(1, 1, -1).cpu())          # wav.cpu() synchronises, as in the reference
            for e in timers:
                t_lat += e[0].elapsed_time(e[1]); t_diff += e[1].elapsed_time(e[2]); t_voc += e[2].elapsed_time(e[3])
            self.last_timings = {"ar_ms": ev[0].elapsed_time(ev[1]), "clvp_ms": ev[1].elapsed_time(ev[2]),
                                 "latents_ms": t_lat, "diffusion_ms": t_diff, "vocoder_ms": t_voc,
                                 "device_total_ms": ev[0].elapsed_time(ev[3])}
            if t_red is not None:
                self.last_timings["redaction_ms"] = t_red
        out = res if len(res) > 1 else res[0]
        if return_deterministic_state:
            return out, (seed, text, voice_samples, conditioning_latents)
        return out
