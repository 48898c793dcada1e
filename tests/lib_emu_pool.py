"""TEST INFRASTRUCTURE ONLY — torch-CPU emulation of the per-row start steps (include/ttb.h row_start: the embed, the
decode step's attention, the sampler and the latent capture), of the slot prefixes (ttb_ar_step_store_prefix_cap) and of
ttb_ar_step_set_group_len, layered over tests/lib_emu_stream.py. With row_start=None every entry is the existing
emulation. `install()` installs lib_emu_stream and these entries, `uninstall()` restores the real binding. Never
imported by the product path."""
import torch
import torch.nn.functional as F

import lib_emu
import lib_emu_grouped
import lib_emu_stream


def _v(t, sizes, strides):
    return torch.as_strided(t, sizes, strides, t.storage_offset())


def _clamp(v, lo, hi):
    return min(max(v, lo), hi)


def ar_embed_step(codes, ld_codes, state, mel_emb, mel_pos, B, D, pos_mode, x, row_start=None):
    if row_start is None:
        return lib_emu.ar_embed_step(codes, ld_codes, state, mel_emb, mel_pos, B, D, pos_mode, x)
    cd = _v(codes, (B, ld_codes), (ld_codes, 1))
    xx = _v(x, (B, D), (D, 1))
    for b in range(B):
        j = _clamp(int(state[0]) - int(row_start[b]), 1, ld_codes)
        xx[b] = mel_emb[int(cd[b, j - 1])] + mel_pos[j + 1 if pos_mode else j]


def ar_sample(logits, ld_logits, V, B, uniforms, ld_u, seen, codes, ld_codes, finished, state, temperature, top_k,
              top_p, rep_penalty, stop_token, advance=True, row_start=None):
    """Row b samples column clamp(step - row_start[b], 0, min(ld_codes, ld_u) - 1): the one-row emulation on a
    scratch counter at that column, then the shared counter advances once."""
    if row_start is None:
        return lib_emu.ar_sample(logits, ld_logits, V, B, uniforms, ld_u, seen, codes, ld_codes, finished, state,
                                 temperature, top_k, top_p, rep_penalty, stop_token, advance)
    step = int(state[0])
    for b in range(B):
        one = torch.zeros(64, dtype=torch.int32)
        one[0] = _clamp(step - int(row_start[b]), 0, min(ld_codes, ld_u) - 1)
        row = lambda t, ld: torch.as_strided(t, (1, ld), (ld, 1), t.storage_offset() + b * ld)
        lib_emu.ar_sample(torch.as_strided(logits, (1, V), (V, 1), logits.storage_offset() + b * ld_logits), V, V, 1,
                          row(uniforms, ld_u), ld_u, seen[b:b + 1], row(codes, ld_codes), ld_codes,
                          finished[b:b + 1], one, temperature, top_k, top_p, rep_penalty, stop_token, advance=False)
    if advance:
        state[0] += 1
        state[1] = int(bool(finished[:B].all()))


def ar_capture_latents(x, B, D, g1, b1, g2, b2, state, Nmax, out, ld_row, row_start=None):
    if row_start is None:
        return lib_emu_stream.ar_capture_latents(x, B, D, g1, b1, g2, b2, state, Nmax, out, ld_row)
    xx = _v(x, (B, D), (D, 1))
    y = F.layer_norm(F.layer_norm(xx, (D,), g1, b1, 1e-5), (D,), g2, b2, 1e-5)
    for b in range(B):
        j = int(state[0]) - 1 - int(row_start[b])
        if 0 <= j < Nmax:
            torch.as_strided(out, (D,), (1,), out.storage_offset() + b * ld_row + j * D).copy_(y[b])


def ar_step_store_prefix(qkv, P, H, pkv, cap=None):
    if cap is None:
        return lib_emu.ar_step_store_prefix(qkv, P, H, pkv)
    assert 0 < P <= cap
    D = H * 64
    r = _v(qkv, (P, 3 * D), (3 * D, 1))
    o = _v(pkv, (H, P, 2, 64), (cap * 128, 128, 64, 1))
    o[:, :, 0].copy_(r[:, D:2 * D].reshape(P, H, 64).transpose(0, 1))
    o[:, :, 1].copy_(r[:, 2 * D:].reshape(P, H, 64).transpose(0, 1))


class ArStep(lib_emu_grouped.ArStep):
    """The grouped step with `row_start` (row b at its own step, clamped to [1, Nmax]) and set_group_len (group g
    attends to the first P of its prefix capacity)."""

    def __init__(self, **kw):
        super().__init__(**kw)
        self.glen = {}

    def set_group_len(self, group, P):
        groups = self.kw.get("groups") or [(0, self.kw["B"], self.kw["P"], self.kw["prefix_kv"])]
        assert 0 < P <= groups[group][2]
        self.glen[group] = int(P)

    def _prefix(self, b):
        k = self.kw
        for g, (b0, b1, Pc, pkv) in enumerate(k.get("groups") or [(0, k["B"], k["P"], k["prefix_kv"])]):
            if b0 <= b < b1:
                P = self.glen.get(g, Pc)
                return P, pkv.view(k["L"], k["H"], Pc, 2, 64)[:, :, :P]
        raise AssertionError("row %d is in no group" % b)

    def step(self, phase_mask=0, layer_begin=0, layer_end=0):
        k = self.kw
        rs = k.get("row_start")
        if rs is None:
            return super().step(phase_mask, layer_begin, layer_end)
        B, D, H, L, V, Nmax = k["B"], k["D"], k["H"], k["L"], k["V"], k["Nmax"]
        step = int(k["state"][0])
        js = [_clamp(step - int(rs[b]), 1, Nmax) for b in range(B)]
        ckv = k["cand_kv"].view(L, B, H, Nmax, 2, 64)

        def attend(l, b, qkv):
            _, pkv = self._prefix(b)
            slot = js[b] - 1
            ckv[l, b, :, slot, 0] = qkv[0, D:2 * D].reshape(H, 64)
            ckv[l, b, :, slot, 1] = qkv[0, 2 * D:].reshape(H, 64)
            q = qkv[0, :D].reshape(H, 1, 64).float() * 0.125
            Kc = torch.cat([pkv[l, :, :, 0].float(), ckv[l, b, :, :slot + 1, 0].float()], 1)
            Vc = torch.cat([pkv[l, :, :, 1].float(), ckv[l, b, :, :slot + 1, 1].float()], 1)
            return (torch.softmax(q @ Kc.transpose(-1, -2), -1) @ Vc).reshape(1, D).to(torch.bfloat16)

        if phase_mask == 4:
            assert layer_end == layer_begin + 1
            qkv = k["qkv"].view(B, 3 * D)
            for b in range(B):
                k["o"].view(B, D)[b:b + 1] = attend(layer_begin, b, qkv[b:b + 1])
            return
        assert phase_mask == 0 and layer_end == 0, "the emulation runs whole steps or one attention phase"

        def ln(v, g, bb):
            return F.layer_norm(v, (D,), g, bb, 1e-5)

        def mm(a, w, bias=None):
            y = a.to(torch.bfloat16).float() @ w.float().t()
            return y if bias is None else y + bias
        codes = k["codes"].view(B, k["ld_codes"])
        for b in range(B):
            j = js[b]
            x = (k["mel_emb"][int(codes[b, j - 1])] + k["mel_pos"][j + 1 if k["pos_mode"] else j]).reshape(1, D)
            for l, lw in enumerate(k["layers"]):
                qkv = mm(ln(x, lw["ln1_g"], lw["ln1_b"]), lw["wqkv"], lw["bqkv"]).to(torch.bfloat16)
                x = x + mm(attend(l, b, qkv), lw["wproj"], lw["bproj"])
                hmid = F.gelu(mm(ln(x, lw["ln2_g"], lw["ln2_b"]), lw["wfc"], lw["bfc"]), approximate="tanh")
                x = x + mm(hmid.to(torch.bfloat16), lw["wproj2"], lw["bproj2"])
            hn = ln(ln(x, k["lnf_g"], k["lnf_b"]), k["fn_g"], k["fn_b"])
            k["x"].view(B, D)[b:b + 1] = x
            k["logits"].view(B, V)[b:b + 1] = mm(hn, k["w_head"], k["b_head"])


_ENTRIES = ("ar_embed_step", "ar_sample", "ar_capture_latents", "ar_step_store_prefix", "ArStep")


def install():
    """Monkeypatch tortoise_tts_b200.lib with the emulation (tests only). Returns what uninstall needs."""
    import sys
    import tortoise_tts_b200.lib as real
    saved = lib_emu_stream.install()
    me = sys.modules[__name__]
    for name in _ENTRIES:
        saved.setdefault(name, getattr(real, name))
        setattr(real, name, getattr(me, name))
    return saved


def uninstall(saved):
    lib_emu_stream.uninstall(saved)
