"""ctypes binding of libttb.so (include/ttb.h). Thin: torch tensors in, raw pointers across the C-ABI.

There is NO fallback: if the library is missing or a call fails, this module raises.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libttb.so")

ACT_NONE, ACT_GELU_NEW, ACT_SILU, ACT_GEGLU, ACT_LRELU02, ACT_TANH = 0, 1, 2, 3, 4, 5
ACT_GELU_ERF = 6


class TtbError(RuntimeError):
    pass


class GemmArgs(C.Structure):
    _fields_ = [("A", C.c_void_p), ("W", C.c_void_p), ("bias", C.c_void_p), ("residual", C.c_void_p),
                ("out_f32", C.c_void_p), ("out_bf16", C.c_void_p),
                ("a_bstride", C.c_longlong), ("res_bstride", C.c_longlong), ("outf_bstride", C.c_longlong),
                ("outb_bstride", C.c_longlong),
                ("lda", C.c_int), ("ldr", C.c_int), ("ldo", C.c_int), ("ldob", C.c_int),
                ("rows", C.c_int), ("M", C.c_int), ("N", C.c_int), ("K", C.c_int),
                ("taps", C.c_int), ("pad", C.c_int), ("batch", C.c_int), ("act", C.c_int),
                ("alpha", C.c_float), ("tile_n", C.c_int), ("force_ref", C.c_int), ("splitk", C.c_int), ("cluster", C.c_int), ("variant", C.c_int),
                ("gn_partials", C.c_void_p), ("gn_groups", C.c_int), ("tap_dilation", C.c_int), ("w_static", C.c_int)]


class AttnArgs(C.Structure):
    _fields_ = [("qkv", C.c_void_p), ("out", C.c_void_p), ("bias", C.c_void_p),
                ("nseq", C.c_int), ("T", C.c_int), ("H", C.c_int),
                ("ld", C.c_int), ("ldo", C.c_int), ("k_off", C.c_int), ("v_off", C.c_int),
                ("scale", C.c_float), ("causal", C.c_int),
                ("kv", C.c_void_p), ("kv_v", C.c_void_p), ("kv_headmajor", C.c_int), ("Tk", C.c_int),
                ("out_f32", C.c_void_p), ("lse", C.c_void_p), ("bias_sat", C.c_int), ("head_dim", C.c_int)]


class DiffStepArgs(C.Structure):
    _fields_ = [("model_out", C.c_void_p), ("out_bstride", C.c_longlong), ("ld_out", C.c_int),
                ("x", C.c_void_p), ("x_bf16", C.c_void_p), ("ld_xb", C.c_int),
                ("noise", C.c_void_p), ("tables", C.c_void_p), ("step", C.c_void_p),
                ("S", C.c_int), ("C", C.c_int), ("iters", C.c_int),
                ("cond_free", C.c_int), ("cond_free_k", C.c_float), ("mel_out", C.c_void_p), ("parity_stride", C.c_longlong)]


class ArStepLayer(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("wqkv", "wproj", "wfc", "wproj2", "ln1_g", "ln1_b", "bqkv", "bproj", "ln2_g",
                                          "ln2_b", "bfc", "bproj2")]


class ArStepArgs(C.Structure):
    _fields_ = [("B", C.c_int), ("D", C.c_int), ("H", C.c_int), ("L", C.c_int), ("V", C.c_int), ("P", C.c_int),
                ("Nmax", C.c_int), ("pos_mode", C.c_int),
                ("layers", C.POINTER(ArStepLayer)), ("w_head", C.c_void_p), ("b_head", C.c_void_p),
                ("lnf_g", C.c_void_p), ("lnf_b", C.c_void_p), ("fn_g", C.c_void_p), ("fn_b", C.c_void_p),
                ("mel_emb", C.c_void_p), ("mel_pos", C.c_void_p), ("codes", C.c_void_p), ("ld_codes", C.c_int),
                ("state", C.c_void_p), ("x", C.c_void_p), ("a", C.c_void_p), ("qkv", C.c_void_p), ("o", C.c_void_p),
                ("h", C.c_void_p), ("hn", C.c_void_p), ("part", C.c_void_p), ("logits", C.c_void_p),
                ("prefix_kv", C.c_void_p), ("cand_kv", C.c_void_p), ("tables", C.c_void_p), ("sync", C.c_void_p),
                ("debug_layer_begin", C.c_int), ("debug_layer_end", C.c_int), ("debug_phase_mask", C.c_int),
                ("attn_compact", C.c_int)]


_lib = None

# every symbol include/ttb.h declares (checked by tests/test_capi_symbols.py)
SYMBOLS = [
    "ttb_last_error", "ttb_version", "ttb_device_ok", "ttb_gemm", "ttb_layernorm", "ttb_rmsnorm", "ttb_groupnorm", "ttb_groupnorm_apply", "ttb_act_split_cast", "ttb_interp_linear",
    "ttb_residual_layernorm", "ttb_attention", "ttb_ar_embed_step", "ttb_ar_decode_attention", "ttb_ar_store_prefix", "ttb_ar_sample",
    "ttb_ar_fix_codes", "ttb_embed", "ttb_clvp_rotary", "ttb_clvp_pool", "ttb_clvp_project",
    "ttb_timestep_embedding", "ttb_linear_small", "ttb_interp_nearest", "ttb_diffusion_step", "ttb_counter_add",
    "ttb_transpose_f32", "ttb_cast_pad_bf16", "ttb_broadcast_rows", "ttb_voc_conv1d", "ttb_voc_convt",
    "ttb_voc_lvc_gate", "ttb_voc_to_tokens_bf16", "ttb_debug_gemm_trace",
    "ttb_ar_step_workspace", "ttb_ar_step_setup", "ttb_ar_decode_step", "ttb_ar_step_store_prefix",
    "ttb_audio_resample", "ttb_audio_stft_mel", "ttb_mean_rows", "ttb_equal_linear",
    "ttb_pair_exchange", "ttb_enable_peer_access", "ttb_peer_alloc", "ttb_peer_open", "ttb_peer_close", "ttb_peer_free",
    "ttb_wav2vec_conv0", "ttb_layernorm_act", "ttb_argmax_rows",
]


def load():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise TtbError("libttb.so not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                       "(no CPU/PyTorch fallback exists for the hot path)")
    lib = C.CDLL(LIB_PATH)
    lib.ttb_last_error.restype = C.c_char_p
    for s in SYMBOLS:
        if s != "ttb_last_error":
            getattr(lib, s).restype = C.c_int
    _lib = lib
    return lib


CALLS = 0   # number of C-ABI compute calls issued (each launches >= 1 kernel); graph replays add their captured count


def add_calls(n):
    global CALLS
    CALLS += n


def _chk(rc, what):
    global CALLS
    CALLS += 1
    if rc != 0:
        raise TtbError("%s failed (%d): %s" % (what, rc, load().ttb_last_error().decode()))


def _p(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _bf(t):
    assert t is None or t.dtype == torch.bfloat16, t.dtype
    return t


def _f32(t):
    assert t is None or t.dtype == torch.float32, t.dtype
    return t


# ------------------------------------------------------------------ wrappers
def gemm(A, W, *, M, N, K, bias=None, residual=None, out_f32=None, out_bf16=None, lda=None, rows=None, batch=1,
         a_bstride=0, res_bstride=0, outf_bstride=0, outb_bstride=0, ldr=None, ldo=None, ldob=None, taps=1, pad=0,
         act=ACT_NONE, alpha=1.0, tile_n=0, force_ref=False, splitk=1, cluster=0, variant=0, gn_partials=None, gn_groups=0, tap_dilation=1, w_static=False):
    """See include/ttb.h ttb_gemm. A: bf16 [batch, rows, lda]; W: bf16 [N, taps*K]. `gn_partials` (a groupnorm_scratch
    buffer): the epilogue also leaves the GroupNorm statistics of the output there (consumed by groupnorm_apply)."""
    _bf(A), _bf(W), _f32(bias), _f32(residual), _f32(out_f32), _bf(out_bf16)
    n_out = N // 2 if act == ACT_GEGLU else N
    g = GemmArgs()
    g.A, g.W, g.bias, g.residual = A.data_ptr(), W.data_ptr(), _p(bias).value or 0, _p(residual).value or 0
    g.out_f32, g.out_bf16 = _p(out_f32).value or 0, _p(out_bf16).value or 0
    g.a_bstride, g.res_bstride, g.outf_bstride, g.outb_bstride = a_bstride, res_bstride, outf_bstride, outb_bstride
    g.lda = K if lda is None else lda
    g.ldr = n_out if ldr is None else ldr
    g.ldo = n_out if ldo is None else ldo
    g.ldob = n_out if ldob is None else ldob
    g.rows = M if rows is None else rows
    g.M, g.N, g.K, g.taps, g.pad, g.batch, g.act = M, N, K, taps, pad, batch, act
    g.alpha, g.tile_n, g.force_ref, g.splitk, g.cluster = alpha, tile_n, 1 if force_ref else 0, splitk, cluster
    g.variant = variant
    g.gn_partials, g.gn_groups = _p(_f32(gn_partials)).value or 0, gn_groups
    g.tap_dilation = tap_dilation
    g.w_static = 1 if w_static else 0
    _chk(load().ttb_gemm(C.byref(g), _stream()), "ttb_gemm")


def debug_gemm_trace(buf):
    """buf: int64 cuda tensor with 8 entries per CTA of the traced launches, or None to switch tracing off."""
    load().ttb_debug_gemm_trace(_p(buf))


def layernorm(x, M, D, g1, b1, g2=None, b2=None, out_bf16=None, out_f32=None):
    _chk(load().ttb_layernorm(_p(_f32(x)), M, D, _p(g1), _p(b1), _p(g2), _p(b2), _p(_bf(out_bf16)), _p(_f32(out_f32)),
                              _stream()), "ttb_layernorm")


def residual_layernorm(x, M, D, partials, nsplit, split_stride, bias, g1, b1, g2=None, b2=None, out_bf16=None,
                       out_f32=None):
    _chk(load().ttb_residual_layernorm(_p(_f32(x)), M, D, _p(_f32(partials)), nsplit, C.c_longlong(split_stride),
                                       _p(bias), _p(g1), _p(b1), _p(g2), _p(b2), _p(_bf(out_bf16)), _p(_f32(out_f32)),
                                       _stream()), "ttb_residual_layernorm")


def rmsnorm(x, M, D, g, out_bf16):
    _chk(load().ttb_rmsnorm(_p(_f32(x)), M, D, _p(g), _p(_bf(out_bf16)), _stream()), "ttb_rmsnorm")


def groupnorm_scratch(B, groups, device):
    """Zeroed scratch for ttb_groupnorm (TTB_GROUPNORM_SCRATCH_FLOATS in include/ttb.h)."""
    return torch.zeros(B * groups * (2 * 128 + 2) + 16, dtype=torch.float32, device=device)


def groupnorm(x, B, S, Cc, groups, gamma, beta, partials, scale_shift=None, ss_bstride=0, ss_row=None, ss_row_stride=0,
              silu=False, out_bf16=None, ldo=0, out_f32=None, ldof=0):
    _chk(load().ttb_groupnorm(_p(_f32(x)), B, S, Cc, groups, _p(gamma), _p(beta), _p(scale_shift), ss_bstride,
                              _p(ss_row), ss_row_stride, 1 if silu else 0, _p(partials), _p(_bf(out_bf16)), ldo, _p(_f32(out_f32)), ldof,
                              _stream()), "ttb_groupnorm")


def groupnorm_apply(x, B, S, Cc, groups, gamma, beta, partials, scale_shift=None, ss_bstride=0, ss_row=None,
                    ss_row_stride=0, silu=False, out_bf16=None, ldo=0, out_f32=None, ldof=0):
    """The apply half of groupnorm for an x whose statistics a gemm(..., gn_partials=partials) already produced."""
    _chk(load().ttb_groupnorm_apply(_p(_f32(x)), B, S, Cc, groups, _p(gamma), _p(beta), _p(scale_shift), ss_bstride,
                                    _p(ss_row), ss_row_stride, 1 if silu else 0, _p(partials), _p(_bf(out_bf16)), ldo,
                                    _p(_f32(out_f32)), ldof, _stream()), "ttb_groupnorm_apply")


def attention(qkv, out, *, nseq, T, H, ld, ldo, k_off, v_off, scale, causal=False, bias=None, bias_sat=0, head_dim=0):
    a = AttnArgs()
    a.head_dim = head_dim
    a.bias_sat = int(bias_sat) if bias is not None else 0
    a.qkv, a.out, a.bias = _bf(qkv).data_ptr(), _bf(out).data_ptr(), _p(_f32(bias)).value or 0
    a.nseq, a.T, a.H, a.ld, a.ldo, a.k_off, a.v_off = nseq, T, H, ld, ldo, k_off, v_off
    a.scale, a.causal = scale, 1 if causal else 0
    _chk(load().ttb_attention(C.byref(a), _stream()), "ttb_attention")


def ar_embed_step(codes, ld_codes, state, mel_emb, mel_pos, B, D, pos_mode, x):
    _chk(load().ttb_ar_embed_step(_p(codes), ld_codes, _p(state), _p(mel_emb), _p(mel_pos), B, D, pos_mode, _p(x),
                                  _stream()), "ttb_ar_embed_step")


def ar_decode_attention(qkv, pk, pv, ck, cv, state, B, H, P, Nmax, out, scratch_o, scratch_lse):
    _chk(load().ttb_ar_decode_attention(_p(_bf(qkv)), _p(_bf(pk)), _p(_bf(pv)), _p(_bf(ck)), _p(_bf(cv)), _p(state),
                                        B, H, P, Nmax, _p(_bf(out)), _p(_f32(scratch_o)), _p(_f32(scratch_lse)),
                                        _stream()), "ttb_ar_decode_attention")


def ar_store_prefix(qkv, P, H, pk, pv):
    _chk(load().ttb_ar_store_prefix(_p(_bf(qkv)), P, H, _p(_bf(pk)), _p(_bf(pv)), _stream()), "ttb_ar_store_prefix")


def ar_step_store_prefix(qkv, P, H, pkv):
    _chk(load().ttb_ar_step_store_prefix(_p(_bf(qkv)), P, H, _p(_bf(pkv)), _stream()), "ttb_ar_step_store_prefix")


AR_STEP_MAX_B, AR_STEP_MAX_P, AR_STEP_MAX_D = 256, 352, 1024    # limits of csrc/ar_step.cu (make_plan)


def ar_step_supported(B, D, H, P):
    return 0 < B <= AR_STEP_MAX_B and 0 < P <= AR_STEP_MAX_P and D == 64 * H and D % 128 == 0 and D <= AR_STEP_MAX_D


class ArStep:
    """Handle of the one-kernel decode step (include/ttb.h TtbArStepArgs): owns the scratch / table / sync buffers and
    keeps every tensor the kernel points at alive. `layers`: list of dicts with the keys of ARWeights.layers."""

    def __init__(self, *, B, D, H, L, V, P, Nmax, pos_mode, layers, w_head, b_head, lnf_g, lnf_b, fn_g, fn_b, mel_emb,
                 mel_pos, codes, ld_codes, state, x, a, qkv, o, h, hn, logits, prefix_kv, cand_kv, attn_compact=False):
        dev = x.device
        self._keep = (layers, w_head, b_head, lnf_g, lnf_b, fn_g, fn_b, mel_emb, mel_pos, codes, state, x, a, qkv, o, h,
                      hn, logits, prefix_kv, cand_kv)
        self._larr = (ArStepLayer * L)()
        for i, lw in enumerate(layers):
            for n in ("wqkv", "wproj", "wfc", "wproj2"):
                setattr(self._larr[i], n, _bf(lw[n]).data_ptr())
            for n in ("ln1_g", "ln1_b", "bqkv", "bproj", "ln2_g", "ln2_b", "bfc", "bproj2"):
                setattr(self._larr[i], n, _f32(lw[n]).data_ptr())
        g = ArStepArgs()
        g.B, g.D, g.H, g.L, g.V, g.P, g.Nmax, g.pos_mode = B, D, H, L, V, P, Nmax, pos_mode
        g.layers = C.cast(self._larr, C.POINTER(ArStepLayer))
        g.w_head, g.b_head = _bf(w_head).data_ptr(), _f32(b_head).data_ptr()
        g.lnf_g, g.lnf_b, g.fn_g, g.fn_b = lnf_g.data_ptr(), lnf_b.data_ptr(), fn_g.data_ptr(), fn_b.data_ptr()
        g.mel_emb, g.mel_pos = _f32(mel_emb).data_ptr(), _f32(mel_pos).data_ptr()
        g.codes, g.ld_codes, g.state = codes.data_ptr(), ld_codes, state.data_ptr()
        g.x, g.a, g.qkv, g.o = _f32(x).data_ptr(), _bf(a).data_ptr(), _bf(qkv).data_ptr(), _bf(o).data_ptr()
        g.h, g.hn, g.logits = _bf(h).data_ptr(), _bf(hn).data_ptr(), _f32(logits).data_ptr()
        g.prefix_kv, g.cand_kv = _bf(prefix_kv).data_ptr(), _bf(cand_kv).data_ptr()
        g.attn_compact = 1 if attn_compact else 0
        pf, tb, sb = C.c_longlong(0), C.c_longlong(0), C.c_longlong(0)
        _chk(load().ttb_ar_step_workspace(C.byref(g), C.byref(pf), C.byref(tb), C.byref(sb)), "ttb_ar_step_workspace")
        self.part = torch.zeros(max(pf.value, 4), dtype=torch.float32, device=dev)
        self.tables = torch.zeros(tb.value, dtype=torch.uint8, device=dev)
        self.sync = torch.zeros(sb.value, dtype=torch.uint8, device=dev)
        g.part, g.tables, g.sync = self.part.data_ptr(), self.tables.data_ptr(), self.sync.data_ptr()
        self.args = g
        _chk(load().ttb_ar_step_setup(C.byref(g), _stream()), "ttb_ar_step_setup")

    def step(self, phase_mask=0, layer_begin=0, layer_end=0):
        """One decode step (all phases by default; phase_mask / layer range select a part, for tests and probes)."""
        g = self.args
        g.debug_phase_mask, g.debug_layer_begin, g.debug_layer_end = phase_mask, layer_begin, layer_end
        _chk(load().ttb_ar_decode_step(C.byref(g), _stream()), "ttb_ar_decode_step")


def ar_sample(logits, ld_logits, V, B, uniforms, ld_u, seen, codes, ld_codes, finished, state, temperature, top_k,
              top_p, rep_penalty, stop_token, advance=True):
    _chk(load().ttb_ar_sample(_p(_f32(logits)), ld_logits, V, B, _p(_f32(uniforms)), ld_u, _p(seen), _p(codes), ld_codes,
                              _p(finished), _p(state), C.c_float(temperature), top_k, C.c_float(top_p),
                              C.c_float(rep_penalty), stop_token, 1 if advance else 0, _stream()), "ttb_ar_sample")


def ar_fix_codes(codes, B, L, stop_token, trim_len):
    _chk(load().ttb_ar_fix_codes(_p(codes), B, L, stop_token, _p(trim_len), _stream()), "ttb_ar_fix_codes")


def embed(ids, pos, n, D, table, pos_table, out):
    _chk(load().ttb_embed(_p(ids), _p(pos), n, D, _p(_f32(table)), _p(_f32(pos_table)), _p(_f32(out)), _stream()),
         "ttb_embed")


def clvp_rotary(qkv, nseq, T, H):
    _chk(load().ttb_clvp_rotary(_p(_bf(qkv)), nseq, T, H, _stream()), "ttb_clvp_rotary")


def clvp_pool(x, nseq, T, D, g, b, out):
    _chk(load().ttb_clvp_pool(_p(_f32(x)), nseq, T, D, _p(g), _p(b), _p(_f32(out)), _stream()), "ttb_clvp_pool")


def clvp_project(pooled, n, D, W, latents, text_latent, temp_exp, scores):
    _chk(load().ttb_clvp_project(_p(_f32(pooled)), n, D, _p(_f32(W)), _p(latents), _p(text_latent),
                                 C.c_float(temp_exp), _p(scores), _stream()), "ttb_clvp_project")


def timestep_embedding(t, n, Cc, out):
    _chk(load().ttb_timestep_embedding(_p(t), n, Cc, _p(_f32(out)), _stream()), "ttb_timestep_embedding")


def linear_small(x, M, K, W, b, N, out, silu_in=False, silu_out=False):
    _chk(load().ttb_linear_small(_p(_f32(x)), M, K, _p(_f32(W)), _p(b), N, 1 if silu_in else 0, 1 if silu_out else 0,
                                 _p(_f32(out)), _stream()), "ttb_linear_small")


def interp_nearest(x, N, S, Cc, out_bf16=None, ldo=0, out_f32=None, ldof=0):
    _chk(load().ttb_interp_nearest(_p(_f32(x)), N, S, Cc, _p(_bf(out_bf16)), ldo, _p(_f32(out_f32)), ldof, _stream()),
         "ttb_interp_nearest")


def pair_exchange(src, local_area, peer_area, n, parity_stride, branch_off, peer_flags, my_flags, counter, epoch, done_ctr,
                  err):
    _chk(load().ttb_pair_exchange(_p(_f32(src)), _p(_f32(local_area)), _p(_f32(peer_area)), C.c_longlong(n),
                                  C.c_longlong(parity_stride), C.c_longlong(branch_off), _p(peer_flags), _p(my_flags),
                                  _p(counter), _p(epoch), _p(done_ctr), _p(err), _stream()), "ttb_pair_exchange")


class RawBuffer:
    """A device buffer that is not a torch tensor (own cudaMalloc allocation or a CUDA-IPC mapping of the partner's):
    quacks enough like a tensor for the wrappers of this module (data_ptr / dtype / is_cuda)."""

    def __init__(self, ptr, dtype, numel, owned):
        self.ptr, self.dtype, self.n, self.owned, self.is_cuda = int(ptr), dtype, int(numel), owned, True

    def data_ptr(self):
        return self.ptr


def peer_alloc(nbytes, dtype):
    """-> (RawBuffer, 64-byte IPC handle)."""
    ptr = C.c_void_p(0)
    h = C.create_string_buffer(64)
    _chk(load().ttb_peer_alloc(C.c_longlong(nbytes), C.byref(ptr), h), "ttb_peer_alloc")
    return RawBuffer(ptr.value, dtype, nbytes // 4, True), h.raw


def peer_open(handle, dtype, numel):
    ptr = C.c_void_p(0)
    _chk(load().ttb_peer_open(C.create_string_buffer(handle, 64), C.byref(ptr)), "ttb_peer_open")
    return RawBuffer(ptr.value, dtype, numel, False)


def enable_peer_access(peer_device):
    _chk(load().ttb_enable_peer_access(int(peer_device)), "ttb_enable_peer_access")


def diffusion_step(model_out, out_bstride, ld_out, x, x_bf16, ld_xb, noise, tables, step, S, Cc, iters, cond_free,
                   cond_free_k, mel_out=None, parity_stride=0):
    a = DiffStepArgs()
    a.parity_stride = parity_stride
    a.model_out, a.out_bstride, a.ld_out = _f32(model_out).data_ptr(), out_bstride, ld_out
    a.x, a.x_bf16, a.ld_xb = _f32(x).data_ptr(), _p(_bf(x_bf16)).value or 0, ld_xb
    a.noise, a.tables, a.step = _f32(noise).data_ptr(), _f32(tables).data_ptr(), step.data_ptr()
    a.S, a.C, a.iters, a.cond_free, a.cond_free_k = S, Cc, iters, 1 if cond_free else 0, cond_free_k
    a.mel_out = _p(_f32(mel_out)).value or 0
    _chk(load().ttb_diffusion_step(C.byref(a), _stream()), "ttb_diffusion_step")


def counter_add(counter, delta):
    _chk(load().ttb_counter_add(_p(counter), delta, _stream()), "ttb_counter_add")


def transpose_f32(inp, R, Cc, out):
    _chk(load().ttb_transpose_f32(_p(_f32(inp)), R, Cc, _p(_f32(out)), _stream()), "ttb_transpose_f32")


def cast_pad_bf16(inp, R, Cc, ld_in, out, ldo, ncols_out=None):
    _chk(load().ttb_cast_pad_bf16(_p(_f32(inp)), R, Cc, ld_in, _p(_bf(out)), ldo, ldo if ncols_out is None else ncols_out,
                                  _stream()), "ttb_cast_pad_bf16")


def broadcast_rows(row, R, Cc, out_f32, out_bf16, ldo):
    _chk(load().ttb_broadcast_rows(_p(_f32(row)), R, Cc, _p(_f32(out_f32)), _p(_bf(out_bf16)), ldo, _stream()),
         "ttb_broadcast_rows")


def audio_resample(x, n, kernels, down, up, klen, width, out, m):
    _chk(load().ttb_audio_resample(_p(_f32(x)), n, _p(_f32(kernels)), down, up, klen, width, _p(_f32(out)), m, _stream()),
         "ttb_audio_resample")


def audio_stft_mel(x, n, n_fft, hop, window, twiddle, fb, n_mels, power, clip, floor_v, div, out_bf16=None, ldo=0,
                   out_f32=None):
    _chk(load().ttb_audio_stft_mel(_p(_f32(x)), n, n_fft, hop, _p(_f32(window)), _p(_f32(twiddle)), _p(_f32(fb)), n_mels,
                                   power, 1 if clip else 0, C.c_float(floor_v), _p(_f32(div)), _p(_bf(out_bf16)), ldo,
                                   _p(_f32(out_f32)), _stream()), "ttb_audio_stft_mel")


def act_split_cast(a, R, Cc, out, ldo, b=None, c=None, scale=1.0, slope=1.0):
    """out bf16 [R, ldo] = [hi | lo | hi | 0...] of leaky_relu((a + b + c) * scale, slope); see include/ttb.h."""
    _chk(load().ttb_act_split_cast(_p(_f32(a)), _p(_f32(b)), _p(_f32(c)), C.c_float(scale), C.c_float(slope), R, Cc,
                                   _p(_bf(out)), ldo, _stream()), "ttb_act_split_cast")


def interp_linear(x, N, Cc, rscale, S, out):
    _chk(load().ttb_interp_linear(_p(_f32(x)), N, Cc, C.c_float(rscale), S, _p(_f32(out)), _stream()), "ttb_interp_linear")


def mean_rows(x, R, Cc, ld, scale, out, accumulate=False):
    _chk(load().ttb_mean_rows(_p(_f32(x)), R, Cc, ld, C.c_float(scale), 1 if accumulate else 0, _p(_f32(out)), _stream()),
         "ttb_mean_rows")


def equal_linear(x, K, W, b, N, out, wscale=1.0, bscale=1.0, slope=1.0, gain=1.0):
    _chk(load().ttb_equal_linear(_p(_f32(x)), K, _p(_f32(W)), _p(_f32(b)), N, C.c_float(wscale), C.c_float(bscale),
                                 C.c_float(slope), C.c_float(gain), _p(_f32(out)), _stream()), "ttb_equal_linear")


def voc_conv1d(x, Cin, L, w, b, Cout, ksize, out, dilation=1, reflect=False, lrelu_in=1.0, lrelu_out=1.0,
               tanh_out=False, residual=None):
    _chk(load().ttb_voc_conv1d(_p(_f32(x)), Cin, L, _p(_f32(w)), _p(b), Cout, ksize, dilation, 1 if reflect else 0,
                               C.c_float(lrelu_in), C.c_float(lrelu_out), 1 if tanh_out else 0, _p(residual),
                               _p(_f32(out)), _stream()), "ttb_voc_conv1d")


def voc_convt(x, Cc, L, w, b, stride, lrelu_in, out):
    _chk(load().ttb_voc_convt(_p(_f32(x)), Cc, L, _p(_f32(w)), _p(b), stride, C.c_float(lrelu_in), _p(_f32(out)),
                              _stream()), "ttb_voc_convt")


def voc_lvc_gate(y, Cc, L, hop, kernels, ldk, koff, bias, ldb, boff, x):
    _chk(load().ttb_voc_lvc_gate(_p(_f32(y)), Cc, L, hop, _p(_f32(kernels)), ldk, koff, _p(_f32(bias)), ldb, boff,
                                 _p(_f32(x)), _stream()), "ttb_voc_lvc_gate")


def voc_to_tokens_bf16(x, Cc, L, out, ldo, split=False):
    _chk(load().ttb_voc_to_tokens_bf16(_p(_f32(x)), Cc, L, _p(_bf(out)), ldo, 1 if split else 0, _stream()),
         "ttb_voc_to_tokens_bf16")


def wav2vec_conv0(x, n, w, b, g, beta, Cc, stats, out, ldo):
    """Clip normalisation + wav2vec2 feature-extractor conv layer 0 + LayerNorm + GELU (include/ttb.h)."""
    _chk(load().ttb_wav2vec_conv0(_p(_f32(x)), n, _p(_f32(w)), _p(_f32(b)), _p(_f32(g)), _p(_f32(beta)), Cc,
                                  _p(_f32(stats)), _p(_bf(out)), ldo, _stream()), "ttb_wav2vec_conv0")


def layernorm_act(x, M, D, g, b, gelu=False, out_bf16=None, out_f32=None):
    _chk(load().ttb_layernorm_act(_p(_f32(x)), M, D, _p(_f32(g)), _p(_f32(b)), 1 if gelu else 0, _p(_bf(out_bf16)),
                                  _p(_f32(out_f32)), _stream()), "ttb_layernorm_act")


def argmax_rows(x, T, V, out):
    assert out.dtype == torch.int32, out.dtype
    _chk(load().ttb_argmax_rows(_p(_f32(x)), T, V, _p(out), _stream()), "ttb_argmax_rows")
