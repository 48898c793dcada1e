"""TEST INFRASTRUCTURE ONLY — torch-CPU emulation of ttb_ar_sample_params (include/ttb.h: the sampler with every row's
settings read from a TtbSampleParams table), row by row over oracle.ar.sample_step and tests/typical_oracle.py, with the
row_start clamp rule of tests/lib_emu_pool.py. `install()` installs lib_emu_pool, the typical entry of
lib_emu_typical and this entry; `uninstall()` restores the real binding. Never imported by the product path."""
import torch

import lib_emu
import lib_emu_pool
import lib_emu_typical
import typical_oracle


def decode_params(params, B):
    """The first B rows of a sample_params_table as dicts (temperature, top_k, top_p, rep_penalty, typical_mass)."""
    f = params[:B, :4].contiguous().view(torch.float32)
    return [dict(temperature=float(f[b, 0]), top_p=float(f[b, 1]), rep_penalty=float(f[b, 2]),
                 typical_mass=float(f[b, 3]), top_k=min(max(int(params[b, 4]), 1), 50)) for b in range(B)]


def ar_sample_params(logits, ld_logits, V, B, uniforms, ld_u, seen, codes, ld_codes, finished, state, params, stop_token,
                     advance=True, row_start=None):
    """Row b samples column step (or clamp(step - row_start[b], 0, min(ld_codes, ld_u) - 1)) with the settings of
    params[b]: the scalar sampler when its typical_mass is 0, the typical one otherwise. The counter advances once."""
    step = int(state[0])
    cd = lib_emu._v(codes, (B, ld_codes), (ld_codes, 1))
    for b, p in enumerate(decode_params(params, B)):
        col = step if row_start is None else min(max(step - int(row_start[b]), 0), min(ld_codes, ld_u) - 1)
        if int(finished[b]):
            cd[b, col] = stop_token
            continue
        row = torch.as_strided(logits, (V,), (1,), logits.storage_offset() + b * ld_logits)
        prev = [w * 32 + bit for w in range(seen.shape[1]) for bit in range(32) if (int(seen[b, w]) >> bit) & 1]
        u = float(uniforms.reshape(-1)[b * ld_u + col])
        if p["typical_mass"] > 0.0:
            tok, _, _ = typical_oracle.sample_step(row, prev, u, p["temperature"], p["top_k"], p["top_p"],
                                                   p["rep_penalty"], p["typical_mass"])
        else:
            from oracle.ar import sample_step
            tok, _, _ = sample_step(row, prev, u, p["temperature"], p["top_k"], p["top_p"], p["rep_penalty"])
        cd[b, col] = tok
        w, bit = divmod(tok, 32)
        seen[b, w] = int(seen[b, w]) | ((1 << bit) if bit < 31 else -(1 << 31))
        if tok == stop_token:
            finished[b] = 1
    if advance:
        state[0] += 1
        state[1] = int(bool(finished[:B].all()))


def install():
    """Monkeypatch tortoise_tts_b200.lib with the stream pool's emulation, ar_sample_typical and ar_sample_params (tests
    only). Returns what uninstall needs."""
    import tortoise_tts_b200.lib as real
    saved = lib_emu_pool.install()
    for name, fn in (("ar_sample_typical", lib_emu_typical.ar_sample_typical), ("ar_sample_params", ar_sample_params)):
        saved.setdefault(name, getattr(real, name))
        setattr(real, name, fn)
    return saved


def uninstall(saved):
    lib_emu_pool.uninstall(saved)
