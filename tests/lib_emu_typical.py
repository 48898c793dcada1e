"""TEST INFRASTRUCTURE ONLY — torch-CPU emulation of ttb_ar_sample_typical (csrc/ar.cu, the TYPICAL instantiation of
ar_sample_kernel), layered over tests/lib_emu.py: `install()` installs lib_emu and then this entry, `uninstall()`
restores the real binding. Never imported by the product path."""
import torch

import lib_emu
import typical_oracle


def ar_sample_typical(logits, ld_logits, V, B, uniforms, ld_u, seen, codes, ld_codes, finished, state, temperature,
                      top_k, top_p, rep_penalty, stop_token, typical_mass, advance=True):
    if not 0.0 < float(typical_mass) <= 1.0:
        raise _error("ttb_ar_sample_typical: typical_mass=%g outside (0, 1]" % typical_mass)
    step = int(state[0])
    cd = lib_emu._v(codes, (B, ld_codes), (ld_codes, 1))
    for b in range(B):
        if int(finished[b]):
            cd[b, step] = stop_token
            continue
        row = torch.as_strided(logits, (V,), (1,), logits.storage_offset() + b * ld_logits)
        prev = [w * 32 + bit for w in range(seen.shape[1]) for bit in range(32) if (int(seen[b, w]) >> bit) & 1]
        tok, _, _ = typical_oracle.sample_step(row, prev, float(uniforms.reshape(-1)[b * ld_u + step]), temperature,
                                               top_k, top_p, rep_penalty, typical_mass)
        cd[b, step] = tok
        w, bit = divmod(tok, 32)
        seen[b, w] = int(seen[b, w]) | ((1 << bit) if bit < 31 else -(1 << 31))
        if tok == stop_token:
            finished[b] = 1
    if advance:
        state[0] += 1
        state[1] = int(bool(finished.all()))


def _error(msg):
    import tortoise_tts_b200.lib as real
    return real.TtbError(msg)


def install():
    """Monkeypatch tortoise_tts_b200.lib with lib_emu and this entry (tests only). Returns what uninstall needs."""
    import tortoise_tts_b200.lib as real
    saved = lib_emu.install()
    saved.setdefault("ar_sample_typical", real.ar_sample_typical)
    real.ar_sample_typical = ar_sample_typical
    return saved


def uninstall(saved):
    lib_emu.uninstall(saved)
