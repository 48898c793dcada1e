"""TEST INFRASTRUCTURE ONLY — torch-CPU emulation of the libttb.so entries of the wav2vec2 aligner (csrc/wav2vec.cu) and
of the exact-GELU GEMM epilogue (TTB_ACT_GELU_ERF), layered over tests/lib_emu.py: `install()` installs lib_emu and
then these, `uninstall()` restores the real binding. Never imported by the product path."""
import torch
import torch.nn.functional as F

import lib_emu

ACT_GELU_ERF = 6


def _v(t, sizes, strides):
    return torch.as_strided(t, sizes, strides, t.storage_offset())


def gemm(A, W, *, act=lib_emu.ACT_NONE, residual=None, out_f32=None, out_bf16=None, M, N, ldr=None, ldo=None,
         ldob=None, res_bstride=0, outf_bstride=0, outb_bstride=0, batch=1, **kw):
    """lib_emu.gemm plus TTB_ACT_GELU_ERF: exact GELU after the bias, before the residual add."""
    if act != ACT_GELU_ERF:
        return lib_emu.gemm(A, W, act=act, residual=residual, out_f32=out_f32, out_bf16=out_bf16, M=M, N=N, ldr=ldr,
                            ldo=ldo, ldob=ldob, res_bstride=res_bstride, outf_bstride=outf_bstride,
                            outb_bstride=outb_bstride, batch=batch, **kw)
    y = torch.empty(batch, M, N)
    lib_emu.gemm(A, W, M=M, N=N, out_f32=y, outf_bstride=M * N, batch=batch, **kw)
    y = F.gelu(y)
    if residual is not None:
        y = y + _v(residual, (batch, M, N), (res_bstride, ldr or N, 1))
    if out_f32 is not None:
        _v(out_f32, (batch, M, N), (outf_bstride, ldo or N, 1)).copy_(y)
    if out_bf16 is not None:
        _v(out_bf16, (batch, M, N), (outb_bstride, ldob or N, 1)).copy_(y.to(torch.bfloat16))


def wav2vec_conv0(x, n, w, b, g, beta, Cc, stats, out, ldo):
    xx = x[:n].double()
    mean, sd = xx.mean(), torch.sqrt(xx.var().float() + 1e-7)
    stats[0], stats[1] = mean.float(), sd
    xn = (x[:n] - mean.float()) / sd
    y = F.conv1d(xn.reshape(1, 1, -1), w.reshape(Cc, 1, 10), b, stride=5)[0].t()
    _v(out, (y.shape[0], Cc), (ldo, 1)).copy_(F.gelu(F.layer_norm(y, (Cc,), g, beta, 1e-5)).to(torch.bfloat16))


def layernorm_act(x, M, D, g, b, gelu=False, out_bf16=None, out_f32=None):
    y = F.layer_norm(_v(x, (M, D), (D, 1)), (D,), g, b, 1e-5)
    if gelu:
        y = F.gelu(y)
    if out_bf16 is not None:
        _v(out_bf16, (M, D), (D, 1)).copy_(y.to(torch.bfloat16))
    if out_f32 is not None:
        _v(out_f32, (M, D), (D, 1)).copy_(y)


def argmax_rows(x, T, V, out):
    out[:T].copy_(_v(x, (T, V), (V, 1)).argmax(-1).to(torch.int32))


def install():
    """Monkeypatch tortoise_tts_b200.lib with lib_emu and these entries (tests only). Returns what uninstall needs."""
    import tortoise_tts_b200.lib as real
    saved = lib_emu.install()
    for name, fn in (("gemm", gemm), ("wav2vec_conv0", wav2vec_conv0), ("layernorm_act", layernorm_act),
                     ("argmax_rows", argmax_rows)):
        saved.setdefault(name, getattr(real, name))
        setattr(real, name, fn)
    return saved


def uninstall(saved):
    lib_emu.uninstall(saved)
