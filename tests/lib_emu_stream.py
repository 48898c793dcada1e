"""TEST INFRASTRUCTURE ONLY — torch-CPU emulation of ttb_ar_capture_latents (include/ttb.h), layered over
tests/lib_emu_grouped.py: `install()` installs lib_emu, the grouped ArStep and this entry, `uninstall()` restores the real
binding. With it the host tests run AREngine.generate_grouped_stream and api_fast.tts_stream_batch on the CPU. Never
imported by the product path."""
import torch
import torch.nn.functional as F

import lib_emu_grouped


def ar_capture_latents(x, B, D, g1, b1, g2, b2, state, Nmax, out, ld_row):
    """out[b * ld_row + (step - 1) * D + c] = final_norm(ln_f(x[b]))[c]: the kernel runs after the sampler, which has
    already advanced the step counter."""
    j = int(state[0]) - 1
    if not 0 <= j < Nmax:
        return
    xx = torch.as_strided(x, (B, D), (D, 1), x.storage_offset())
    y = F.layer_norm(F.layer_norm(xx, (D,), g1, b1, 1e-5), (D,), g2, b2, 1e-5)
    torch.as_strided(out, (B, D), (ld_row, 1), out.storage_offset() + j * D).copy_(y)


def install():
    """Monkeypatch tortoise_tts_b200.lib with the emulation (tests only). Returns what uninstall needs."""
    import tortoise_tts_b200.lib as real
    saved = lib_emu_grouped.install()
    saved["ar_capture_latents"] = real.ar_capture_latents
    real.ar_capture_latents = ar_capture_latents
    return saved


def uninstall(saved):
    lib_emu_grouped.uninstall(saved)
