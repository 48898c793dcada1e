"""TEST INFRASTRUCTURE ONLY — torch-CPU emulation of the one-kernel decode step with prompt groups (csrc/ar_step.cu,
TtbArStepArgs.groups), layered over tests/lib_emu.py: `install()` installs lib_emu and then this ArStep, `uninstall()`
restores the real binding. Every row is computed on its own (one-row matmuls), so a row's result does not depend on
which other rows share its batch: the kernels are row-independent, and so is this emulation. Never imported by the
product path."""
import torch
import torch.nn.functional as F

import lib_emu


class ArStep(lib_emu.ArStep):
    """lib.ArStep with `groups` = [(row_begin, row_end, P, prefix_kv), ...] (None: every row attends to prefix_kv)."""

    def _prefix(self, b):
        k = self.kw
        for b0, b1, P, pkv in (k.get("groups") or [(0, k["B"], k["P"], k["prefix_kv"])]):
            if b0 <= b < b1:
                return P, pkv.view(k["L"], k["H"], P, 2, 64)
        raise AssertionError("row %d is in no group" % b)

    def step(self, phase_mask=0, layer_begin=0, layer_end=0):
        k = self.kw
        B, D, H, L, V, Nmax = k["B"], k["D"], k["H"], k["L"], k["V"], k["Nmax"]
        j = int(k["state"][0])
        slot = j - 1
        ckv = k["cand_kv"].view(L, B, H, Nmax, 2, 64)

        def attend(l, b, qkv):                        # qkv [1, 3D] bf16 -> o [1, D] bf16, with the KV append
            _, pkv = self._prefix(b)
            ckv[l, b, :, slot, 0] = qkv[0, D:2 * D].reshape(H, 64)
            ckv[l, b, :, slot, 1] = qkv[0, 2 * D:].reshape(H, 64)
            q = qkv[0, :D].reshape(H, 1, 64).float() * 0.125
            Kc = torch.cat([pkv[l, :, :, 0].float(), ckv[l, b, :, :slot + 1, 0].float()], 1)
            Vc = torch.cat([pkv[l, :, :, 1].float(), ckv[l, b, :, :slot + 1, 1].float()], 1)
            return (torch.softmax(q @ Kc.transpose(-1, -2), -1) @ Vc).reshape(1, D).to(torch.bfloat16)

        if phase_mask == 4:          # attention phase of one layer (the "mixed" mode of AREngine)
            assert layer_end == layer_begin + 1
            qkv = k["qkv"].view(B, 3 * D)
            for b in range(B):
                k["o"].view(B, D)[b:b + 1] = attend(layer_begin, b, qkv[b:b + 1])
            return
        assert phase_mask == 0 and layer_end == 0, "the emulation runs whole steps or one attention phase"

        def ln(v, g, bb):
            return F.layer_norm(v, (D,), g, bb, 1e-5)

        def mm(a, w, bias=None):                    # bf16 operands, fp32 accumulate
            y = a.to(torch.bfloat16).float() @ w.float().t()
            return y if bias is None else y + bias
        codes = k["codes"].view(B, k["ld_codes"])
        for b in range(B):
            tok = int(codes[b, j - 1])
            x = (k["mel_emb"][tok] + k["mel_pos"][j + 1 if k["pos_mode"] else j]).reshape(1, D)
            for l, lw in enumerate(k["layers"]):
                qkv = mm(ln(x, lw["ln1_g"], lw["ln1_b"]), lw["wqkv"], lw["bqkv"]).to(torch.bfloat16)
                x = x + mm(attend(l, b, qkv), lw["wproj"], lw["bproj"])
                hmid = F.gelu(mm(ln(x, lw["ln2_g"], lw["ln2_b"]), lw["wfc"], lw["bfc"]), approximate="tanh")
                x = x + mm(hmid.to(torch.bfloat16), lw["wproj2"], lw["bproj2"])
            hn = ln(ln(x, k["lnf_g"], k["lnf_b"]), k["fn_g"], k["fn_b"])
            k["x"].view(B, D)[b:b + 1] = x
            k["logits"].view(B, V)[b:b + 1] = mm(hn, k["w_head"], k["b_head"])


def install():
    """Monkeypatch tortoise_tts_b200.lib with lib_emu and this ArStep (tests only). Returns what uninstall needs."""
    import tortoise_tts_b200.lib as real
    saved = lib_emu.install()
    real.ArStep = ArStep
    return saved


def uninstall(saved):
    lib_emu.uninstall(saved)
