"""TEST INFRASTRUCTURE ONLY — loader for the unmodified reference (neonbjb/tortoise-tts).

Imports the reference's own PyTorch modules from a checkout of the reference (TORTOISE_REFERENCE_ROOT) or, where
there is none, from the copy that oracle/build_ref.py placed under oracle/_ref, so that (a) oracle/*.py restatements can be
validated against them and (b) golden vectors under tests/golden/ can be generated
(tests/golden/make_golden.py).  Nothing in the product path may import this file.

Shims follow SURVEY.md App. C-1: the image has transformers 5.x while the reference
pins 4.31, and several pure-host dependencies (librosa, inflect, ...) are absent.
"""
import os
import sys
import types

_VENDORED = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")    # oracle/build_ref.py (git-ignored copy)
REFERENCE_ROOT = os.environ.get("TORTOISE_REFERENCE_ROOT", "/root/reference")
if not os.path.isdir(os.path.join(REFERENCE_ROOT, "tortoise")) and os.path.isdir(os.path.join(_VENDORED, "tortoise")):
    REFERENCE_ROOT = _VENDORED                # the unmodified reference package as copied by the build recipe


def reference_available() -> bool:
    return os.path.isdir(os.path.join(REFERENCE_ROOT, "tortoise"))


_loaded = False


def load_reference():
    """Import the reference package with the shims applied. Returns the `tortoise` module."""
    global _loaded
    if not reference_available():
        raise RuntimeError("reference not present at %s" % REFERENCE_ROOT)
    if _loaded:
        import tortoise
        return tortoise

    def stub(name, **attrs):
        m = types.ModuleType(name)
        for k, v in attrs.items():
            setattr(m, k, v)
        sys.modules[name] = m
        return m

    # transformers must be imported BEFORE stubbing librosa (its lazy module probes find_spec)
    # force the lazy transformers module to materialise before patching (App. C-1)
    import transformers
    from transformers import GPT2Config, GPT2PreTrainedModel, GPT2Model, LogitsProcessor, GenerationMixin  # noqa
    if "transformers.utils.model_parallel_utils" not in sys.modules:
        stub("transformers.utils.model_parallel_utils",
             get_device_map=lambda *a, **k: None, assert_device_map=lambda *a, **k: None)
    for _tm in {id(transformers): transformers, id(sys.modules["transformers"]): sys.modules["transformers"]}.values():
        if "LogitsWarper" not in _tm.__dict__:
            _tm.LogitsWarper = LogitsProcessor

    class _Dummy:
        def __init__(self, *a, **k):
            pass

    if "rotary_embedding_torch" not in sys.modules:
        stub("rotary_embedding_torch", RotaryEmbedding=_Dummy, broadcat=lambda *a, **k: None)
    if "progressbar" not in sys.modules:
        stub("progressbar")

    class _Inflect:
        def number_to_words(self, x, **k):
            return str(x)
    if "inflect" not in sys.modules:
        stub("inflect", engine=lambda: _Inflect())
    if "unidecode" not in sys.modules:
        stub("unidecode", unidecode=lambda s: s)
    if "librosa" not in sys.modules:
        lib = stub("librosa")
        lib.util = stub("librosa.util", pad_center=lambda data, size=None, **k: data, tiny=lambda x: 1e-30)
        lib.filters = stub("librosa.filters", mel=None)

    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    import tortoise.models.autoregressive as ar
    if GenerationMixin not in ar.GPT2InferenceModel.__mro__:
        ar.GPT2InferenceModel.__bases__ = ar.GPT2InferenceModel.__bases__ + (GenerationMixin,)
    _loaded = True
    import tortoise
    return tortoise
