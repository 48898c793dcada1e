"""UnifiedVoice autoregressive stage on the sm_90a kernels (hot loop 1 + latents, SURVEY §8 rows a1-a4, a7).

Host side mirrors `UnifiedVoice.inference_speech` / `UnifiedVoice.forward(return_latent=True)`
(tortoise/models/autoregressive.py:535-563, 454-512): same inputs (conditioning latent, zero-padded text
tokens), same outputs (codes / latents). All arithmetic runs in libttb.so; torch is used for allocation,
weight packing at load time, and CUDA-graph capture of the decode step.
"""
import torch

from . import lib
from .config import ModelConfig


def _bf(t, dev):
    return t.to(device=dev, dtype=torch.bfloat16).contiguous()


def _f(t, dev):
    return t.to(device=dev, dtype=torch.float32).contiguous()


class ARWeights:
    """Packs `autoregressive.pth` (SURVEY App. B): HF Conv1D weights [in,out] are transposed to K-major bf16."""

    def __init__(self, sd, cfg: ModelConfig, dev):
        D = cfg.ar_dim
        self.layers = []
        for l in range(cfg.ar_layers):
            p = f"gpt.h.{l}."
            self.layers.append(dict(
                ln1_g=_f(sd[p + "ln_1.weight"], dev), ln1_b=_f(sd[p + "ln_1.bias"], dev),
                wqkv=_bf(sd[p + "attn.c_attn.weight"].t(), dev), bqkv=_f(sd[p + "attn.c_attn.bias"], dev),
                wproj=_bf(sd[p + "attn.c_proj.weight"].t(), dev), bproj=_f(sd[p + "attn.c_proj.bias"], dev),
                ln2_g=_f(sd[p + "ln_2.weight"], dev), ln2_b=_f(sd[p + "ln_2.bias"], dev),
                wfc=_bf(sd[p + "mlp.c_fc.weight"].t(), dev), bfc=_f(sd[p + "mlp.c_fc.bias"], dev),
                wproj2=_bf(sd[p + "mlp.c_proj.weight"].t(), dev), bproj2=_f(sd[p + "mlp.c_proj.bias"], dev)))
        self.lnf_g, self.lnf_b = _f(sd["gpt.ln_f.weight"], dev), _f(sd["gpt.ln_f.bias"], dev)
        self.fn_g, self.fn_b = _f(sd["final_norm.weight"], dev), _f(sd["final_norm.bias"], dev)
        self.text_emb = _f(sd["text_embedding.weight"], dev)
        self.mel_emb = _f(sd["mel_embedding.weight"], dev)
        self.mel_pos = _f(sd["mel_pos_embedding.emb.weight"], dev)
        self.text_pos = _f(sd["text_pos_embedding.emb.weight"], dev)
        self.w_head = _bf(sd["mel_head.weight"], dev)
        self.b_head = _f(sd["mel_head.bias"], dev)


class AREngine:
    def __init__(self, sd, cfg: ModelConfig, device="cuda"):
        self.cfg = cfg
        self.dev = torch.device(device)
        self.w = ARWeights(sd, cfg, self.dev)
        self.D = cfg.ar_dim
        self.H = cfg.ar_heads
        self.V = cfg.number_mel_codes
        self._dec = None  # decode workspace keyed by (B, P, Nmax)

    import os as _os
    DECODE_CLUSTER = int(_os.environ.get("TTB_AR_CLUSTER", "0"))
    # TTB_AR_WIDE=1: c_attn / c_fc (N = 3D, 4D: one wave of 64-wide tiles) use 64-column tiles with an 8-stage pipeline
    DECODE_WIDE = int(_os.environ.get("TTB_AR_WIDE", "0"))
    # TTB_AR_FUSED=1 (default): the decode step is ONE persistent kernel (csrc/ar_step.cu) + the sampler; 0 = the
    # per-op CUDA graph (kept as the A/B baseline and for shapes the fused kernel does not cover)
    FUSED = int(_os.environ.get("TTB_AR_FUSED", "1"))
    # How the step runs when the one-kernel form is available: "fused" = everything in the persistent kernel, whose
    # phases grow with the batch (one CTA per SM serialises TMA wait -> MMA -> epilogue inside a phase, which several
    # small kernels per SM overlap). "mixed" = the per-op graph with its three attention kernels (prefix flash + candidate
    # stream + merge) replaced by the persistent kernel's attention phase (one launch). "auto" picks by batch size: the
    # one-kernel step for small batches only (H100 80GB HBM3, 700 W, 256 candidates, 429 steps: AR 1.73 s mixed against
    # 3.50 s fused; the batch size where the two cross, FUSED_MAX_B, has not been measured on H100).
    MODE = _os.environ.get("TTB_AR_MODE", "auto")            # auto | fused | mixed | perop
    FUSED_MAX_B = int(_os.environ.get("TTB_AR_FUSED_MAX_B", "16"))
    # TTB_AR_CHAINS=2: in mixed mode the candidates are decoded as TWO independent half-batches on two streams inside
    # one captured step. Every kernel of the chain LN -> c_attn -> attention -> c_proj -> LN -> c_fc -> mlp.c_proj is
    # bound by its own latency except the attention (HBM-bound), so the chain of one half fills the bubbles of the
    # other; the attention then runs in compact CTAs (lib.ArStep attn_compact) that leave room for a GEMM CTA per SM.
    # which decode GEMMs may fetch their weights ahead of griddepcontrol.wait (TtbGemmArgs.w_static): "ln" = the ones that
    # follow a LayerNorm (which triggers its dependents early), "all", "none"
    WSTATIC = _os.environ.get("TTB_AR_WSTATIC", "ln")
    # measured on H100 (80GB HBM3, 700 W) at 256 candidates: AR 1839 ms with one chain, 1727 ms with two; split-K 2 / 4
    # against none: 1727 against 1795 ms; weight prefetch ahead of the dependency wait ("ln" against "none"): 1727 / 1731 ms
    # (inside the run-to-run spread). CHAINS_MIN_B has not been measured on H100.
    CHAINS = int(_os.environ.get("TTB_AR_CHAINS", "2"))
    CHAINS_MIN_B = int(_os.environ.get("TTB_AR_CHAINS_MIN_B", "128"))
    SPLITK_PROJ = int(_os.environ.get("TTB_AR_SPLITK_PROJ", "2"))     # attn.c_proj (K = D): 32 n-tiles x 2 m-tiles x 2 splits = 128 CTAs at D=1024, B=256
    SPLITK_PROJ2 = int(_os.environ.get("TTB_AR_SPLITK_PROJ2", "4"))   # mlp.c_proj (K = 4D): 32 x 2 x 4 = 256 CTAs

    @staticmethod
    def _nsplit(kb_total, splitk):
        """Number of K ranges ttb_gemm actually creates for `splitk` requested splits (every split owns >= 1 block)."""
        per = (kb_total + splitk - 1) // splitk
        return (kb_total + per - 1) // per

    # ------------------------------------------------------------------ shared trunk over M tokens
    def _alloc_trunk(self, M):
        D, dev = self.D, self.dev
        return dict(a=torch.empty(M, D, dtype=torch.bfloat16, device=dev),
                    qkv=torch.empty(M, 3 * D, dtype=torch.bfloat16, device=dev),
                    o=torch.empty(M, D, dtype=torch.bfloat16, device=dev),
                    h=torch.empty(M, 4 * D, dtype=torch.bfloat16, device=dev))

    def _layer(self, lw, x, M, ws, attn_fn):
        D = self.D
        lib.layernorm(x, M, D, lw["ln1_g"], lw["ln1_b"], out_bf16=ws["a"])
        lib.gemm(ws["a"], lw["wqkv"], M=M, N=3 * D, K=D, bias=lw["bqkv"], out_bf16=ws["qkv"])
        attn_fn(ws["qkv"], ws["o"])
        lib.gemm(ws["o"], lw["wproj"], M=M, N=D, K=D, bias=lw["bproj"], residual=x, out_f32=x)
        lib.layernorm(x, M, D, lw["ln2_g"], lw["ln2_b"], out_bf16=ws["a"])
        lib.gemm(ws["a"], lw["wfc"], M=M, N=4 * D, K=D, bias=lw["bfc"], act=lib.ACT_GELU_NEW, out_bf16=ws["h"])
        lib.gemm(ws["h"], lw["wproj2"], M=M, N=D, K=4 * D, bias=lw["bproj2"], residual=x, out_f32=x)

    def _prompt_ids(self, text_tokens):
        cfg = self.cfg
        t = [int(v) for v in text_tokens]
        return [cfg.start_text_token] + t + [cfg.stop_text_token]   # autoregressive.py:538-539 (api.py:391 padded once)

    # ------------------------------------------------------------------ prefill
    def _prefill(self, cond_latent, text_tokens, st):
        """Runs the prompt [cond | text(T+3) | start_mel] once (shared by every candidate), fills the prefix
        KV cache and returns logits of the first sampling step [1, V]."""
        cfg, D, H, dev = self.cfg, self.D, self.H, self.dev
        ids = self._prompt_ids(text_tokens)
        P = len(ids) + 2
        assert P == st["P"]
        x = st["px"]
        # rows 1..P-2: text, row P-1: start mel token at mel position 0, row 0: conditioning latent
        tid = torch.tensor(ids, dtype=torch.int32, device=dev)
        tpos = torch.arange(len(ids), dtype=torch.int32, device=dev)
        lib.embed(tid, tpos, len(ids), D, self.w.text_emb, self.w.text_pos, x[1:])
        sid = torch.tensor([cfg.start_mel_token], dtype=torch.int32, device=dev)
        spos = torch.zeros(1, dtype=torch.int32, device=dev)
        lib.embed(sid, spos, 1, D, self.w.mel_emb, self.w.mel_pos, x[P - 1:])
        x[0].copy_(cond_latent.reshape(-1).to(device=dev, dtype=torch.float32))
        ws = st["pws"]
        for l, lw in enumerate(self.w.layers):
            def attn(qkv, o, l=l):
                if st["fused"]:
                    lib.ar_step_store_prefix(qkv, P, H, st["pkv"][l])
                else:
                    lib.ar_store_prefix(qkv, P, H, st["pk"][l], st["pv"][l])
                lib.attention(qkv, o, nseq=1, T=P, H=H, ld=3 * D, ldo=D, k_off=D, v_off=2 * D, scale=0.125, causal=True)
            self._layer(lw, x, P, ws, attn)
        lib.layernorm(x[P - 1:], 1, D, self.w.lnf_g, self.w.lnf_b, self.w.fn_g, self.w.fn_b, out_bf16=st["hn"][:1])
        lib.gemm(st["hn"], self.w.w_head, M=1, N=self.V, K=D, bias=self.w.b_head, out_f32=st["logits"])

    # ------------------------------------------------------------------ decode workspace + graph
    def _decode_state(self, B, P, Nmax):
        key = (B, P, Nmax)
        if self._dec is not None and self._dec["key"] == key:
            return self._dec
        self._dec = None                  # release the previous workspace (KV caches) before allocating the next
        cfg, D, dev = self.cfg, self.D, self.dev
        ok = bool(self.FUSED) and lib.ar_step_supported(B, D, self.H, P)
        mode = self.MODE if ok else "perop"
        if mode == "auto":
            mode = "fused" if B <= self.FUSED_MAX_B else "mixed"
        nch = self.CHAINS if (mode == "mixed" and self.CHAINS > 1 and B >= self.CHAINS_MIN_B and B % self.CHAINS == 0) else 1
        st = dict(key=key, P=P, B=B, Nmax=Nmax, mode=mode, fused=mode in ("fused", "mixed"))
        L, H = cfg.ar_layers, self.H
        # ---- prompt prefill (shared by every candidate and every chain)
        st["px"] = torch.empty(P, D, dtype=torch.float32, device=dev)
        st["pws"] = self._alloc_trunk(P)
        if st["fused"]:
            # K and V of a position adjacent: one (candidate, head) stream is one contiguous byte range (csrc/ar_step.cu)
            st["pkv"] = torch.empty(L, H, P, 2, 64, dtype=torch.bfloat16, device=dev)
        else:
            st["pk"] = torch.empty(L, H, P, 64, dtype=torch.bfloat16, device=dev)
            st["pv"] = torch.empty(L, H, P, 64, dtype=torch.bfloat16, device=dev)
        st["hn"] = torch.empty(1, D, dtype=torch.bfloat16, device=dev)
        st["logits"] = torch.empty(1, self.V, dtype=torch.float32, device=dev)
        # ---- decode workspaces: one per chain (contiguous candidate ranges)
        per = B // nch
        st["chains"] = [self._chain_state(st, per, c * per, compact=nch > 1) for c in range(nch)]
        st["sides"] = [torch.cuda.Stream(device=dev) for _ in range(nch - 1)] if dev.type == "cuda" else []
        st["graph"] = None
        st["graph_params"] = None
        self._dec = st
        return st

    def _chain_state(self, st, B, b0, compact=False):
        """Decode workspace of candidates [b0, b0 + B): residual stream, trunk buffers, candidate KV cache, sampler state."""
        cfg, D, H, dev = self.cfg, self.D, self.H, self.dev
        L, Nmax = cfg.ar_layers, st["Nmax"]
        ch = dict(B=B, b0=b0, P=st["P"], Nmax=Nmax, mode=st["mode"], fused=st["fused"], compact=compact)
        if st["fused"]:
            ch["pkv"] = st["pkv"]
            ch["ckv"] = torch.zeros(L, B, H, Nmax, 2, 64, dtype=torch.bfloat16, device=dev)
        else:
            ch["pk"], ch["pv"] = st["pk"], st["pv"]
            ch["ck"] = torch.zeros(L, B, H, Nmax, 64, dtype=torch.bfloat16, device=dev)
            ch["cv"] = torch.zeros(L, B, H, Nmax, 64, dtype=torch.bfloat16, device=dev)
        ch["x"] = torch.empty(B, D, dtype=torch.float32, device=dev)
        ch["ws"] = self._alloc_trunk(B)
        ch["hn"] = torch.empty(max(B, 1), D, dtype=torch.bfloat16, device=dev)
        ch["att_o"] = torch.zeros(2, B, D, dtype=torch.float32, device=dev)      # [prefix | candidate] partial rows
        ch["att_lse"] = torch.zeros(2, B, H, dtype=torch.float32, device=dev)
        ch["part_a"] = torch.zeros(max(self.SPLITK_PROJ, 2), B, D, dtype=torch.float32, device=dev)
        ch["part_b"] = torch.zeros(max(self.SPLITK_PROJ2, 2), B, D, dtype=torch.float32, device=dev)
        ch["logits"] = torch.empty(B, self.V, dtype=torch.float32, device=dev)
        ch["state"] = torch.zeros(64, dtype=torch.int32, device=dev)
        ch["codes"] = torch.empty(B, Nmax, dtype=torch.int32, device=dev)
        ch["seen"] = torch.zeros(B, (self.V + 31) // 32, dtype=torch.int32, device=dev)
        ch["finished"] = torch.zeros(B, dtype=torch.int32, device=dev)
        ch["uniforms"] = torch.empty(B, Nmax, dtype=torch.float32, device=dev)
        ch["step_handles"] = {}
        return ch

    def _step_handle(self, st, pos_mode):
        """The one-kernel decode step bound to this workspace (tensor maps are built once per workspace + position rule)."""
        hd = st["step_handles"].get(pos_mode)
        if hd is None:
            w, ws = self.w, st["ws"]
            hd = lib.ArStep(B=st["B"], D=self.D, H=self.H, L=self.cfg.ar_layers, V=self.V, P=st["P"], Nmax=st["Nmax"],
                            pos_mode=pos_mode, layers=w.layers, w_head=w.w_head, b_head=w.b_head, lnf_g=w.lnf_g,
                            lnf_b=w.lnf_b, fn_g=w.fn_g, fn_b=w.fn_b, mel_emb=w.mel_emb, mel_pos=w.mel_pos,
                            codes=st["codes"], ld_codes=st["Nmax"], state=st["state"], x=st["x"], a=ws["a"], qkv=ws["qkv"],
                            o=ws["o"], h=ws["h"], hn=st["hn"], logits=st["logits"], prefix_kv=st["pkv"], cand_kv=st["ckv"],
                            attn_compact=bool(st.get("compact")))
            st["step_handles"][pos_mode] = hd
        return hd

    def _decode_step(self, st, sp):
        """One decode step of every chain: chain 0 on the current stream, every other chain on its own side stream (forked
        and joined with events, so the whole step is still ONE capturable unit)."""
        chains = st["chains"]
        if len(chains) == 1 or not st["sides"]:
            for ch in chains:
                self._chain_step(ch, sp)
            return
        cur = torch.cuda.current_stream()
        for side in st["sides"]:
            side.wait_stream(cur)
        self._chain_step(chains[0], sp)
        for ch, side in zip(chains[1:], st["sides"]):
            with torch.cuda.stream(side):
                self._chain_step(ch, sp)
        for side in st["sides"]:
            cur.wait_stream(side)

    def _chain_step(self, st, sp):
        """One trunk pass for the last sampled token of every candidate of one chain + fused sampling of the next one."""
        B, P, Nmax, D, H = st["B"], st["P"], st["Nmax"], self.D, self.H
        x, ws = st["x"], st["ws"]
        if st["mode"] == "fused":
            self._step_handle(st, sp["pos_mode"]).step()
            lib.ar_sample(st["logits"], self.V, self.V, B, st["uniforms"], Nmax, st["seen"], st["codes"], Nmax,
                          st["finished"], st["state"], sp["temperature"], sp["top_k"], sp["top_p"], sp["rep_penalty"],
                          self.cfg.stop_mel_token, advance=True)
            return
        hd = self._step_handle(st, sp["pos_mode"]) if st["mode"] == "mixed" else None
        lib.ar_embed_step(st["codes"], Nmax, st["state"], self.w.mel_emb, self.w.mel_pos, B, D, sp["pos_mode"], x)
        # Skinny-M decode (M = B candidates): every GEMM is weight-streaming bound, so the grid is widened with
        # 32-column tiles and, for the two GEMMs that feed the residual stream, split-K; their partial sums, bias and
        # the residual add are folded into the LayerNorm that follows (fixed summation order -> deterministic).
        kb = D // 64
        # thread-block clusters sharing the activation tile by TMA multicast (TTB_AR_CLUSTER=0 disables)
        cl = self.DECODE_CLUSTER if D % 128 == 0 else 0
        s1 = min(self.SPLITK_PROJ, kb)
        s2 = min(self.SPLITK_PROJ2, 4 * kb)
        pa, pb = st["part_a"], st["part_b"]
        wide = dict(tile_n=64, variant=3) if (self.DECODE_WIDE and not cl) else dict(tile_n=32)
        ws_ln, ws_all = self.WSTATIC in ("ln", "all"), self.WSTATIC == "all"
        prev = None   # (partials, nsplit, bias) of the previous layer's mlp.c_proj, folded into the next LayerNorm
        for l, lw in enumerate(self.w.layers):
            if prev is None:
                lib.layernorm(x, B, D, lw["ln1_g"], lw["ln1_b"], out_bf16=ws["a"])
            else:
                lib.residual_layernorm(x, B, D, prev[0], prev[1], B * D, prev[2], lw["ln1_g"], lw["ln1_b"], out_bf16=ws["a"])
            lib.gemm(ws["a"], lw["wqkv"], M=B, N=3 * D, K=D, bias=lw["bqkv"], out_bf16=ws["qkv"], cluster=cl, w_static=ws_ln,
                     **wide)
            if hd is not None:
                hd.step(phase_mask=4, layer_begin=l, layer_end=l + 1)     # attention phase of the persistent kernel
            else:
                lib.ar_decode_attention(ws["qkv"], st["pk"][l], st["pv"][l], st["ck"][l], st["cv"][l], st["state"], B, H,
                                        P, Nmax, ws["o"], st["att_o"], st["att_lse"])
            lib.gemm(ws["o"], lw["wproj"], M=B, N=D, K=D, out_f32=pa, outf_bstride=B * D, tile_n=32, splitk=max(s1, 2), cluster=cl,
                     w_static=ws_all)
            lib.residual_layernorm(x, B, D, pa, self._nsplit(kb, max(s1, 2)), B * D, lw["bproj"], lw["ln2_g"], lw["ln2_b"],
                                   out_bf16=ws["a"])
            lib.gemm(ws["a"], lw["wfc"], M=B, N=4 * D, K=D, bias=lw["bfc"], act=lib.ACT_GELU_NEW, out_bf16=ws["h"],
                     cluster=cl, w_static=ws_ln, **wide)
            lib.gemm(ws["h"], lw["wproj2"], M=B, N=D, K=4 * D, out_f32=pb, outf_bstride=B * D, tile_n=32, cluster=cl,
                     splitk=max(s2, 2), w_static=ws_all)
            prev = (pb, self._nsplit(4 * kb, max(s2, 2)), lw["bproj2"])
        lib.residual_layernorm(x, B, D, prev[0], prev[1], B * D, prev[2], self.w.lnf_g, self.w.lnf_b, self.w.fn_g,
                               self.w.fn_b, out_bf16=st["hn"])
        lib.gemm(st["hn"], self.w.w_head, M=B, N=self.V, K=D, bias=self.w.b_head, out_f32=st["logits"], w_static=ws_ln)
        lib.ar_sample(st["logits"], self.V, self.V, B, st["uniforms"], Nmax, st["seen"], st["codes"], Nmax,
                      st["finished"], st["state"], sp["temperature"], sp["top_k"], sp["top_p"], sp["rep_penalty"],
                      self.cfg.stop_mel_token, advance=True)

    def _begin(self, cond_latent, text_tokens, B, Nmax, uniforms, seed, sp, trace_logits=None):
        """Workspace reset + prompt prefill + the first sampled token of every candidate."""
        cfg, dev = self.cfg, self.dev
        P = len(text_tokens) + 4  # cond + [start, tokens(padded), stop] + start_mel
        st = self._decode_state(B, P, Nmax)
        if uniforms is None:
            g = torch.Generator(device=dev)
            g.manual_seed(0 if seed is None else int(seed))
            uniforms = torch.rand(B, Nmax, generator=g, device=dev)
        uniforms = uniforms.to(device=dev, dtype=torch.float32)
        self._prefill(cond_latent, text_tokens, st)
        if trace_logits is not None:   # parity hook (eager mode): logits the sampler sees at every step
            trace_logits.append(st["logits"][:1].expand(B, -1).clone())
        w, bit = divmod(cfg.start_mel_token, 32)
        for ch in st["chains"]:
            ch["uniforms"].copy_(uniforms[ch["b0"]: ch["b0"] + ch["B"]])
            ch["state"].zero_()
            ch["finished"].zero_()
            ch["codes"].fill_(cfg.stop_mel_token)
            ch["seen"].zero_()
            # HF's repetition penalty sees the fake prompt ids {1, start_mel} (autoregressive.py:546-548)
            ch["seen"][:, 0] = 2
            ch["seen"][:, w] |= (1 << bit) if bit < 31 else -(1 << 31)
            lib.ar_sample(st["logits"], 0, self.V, ch["B"], ch["uniforms"], Nmax, ch["seen"], ch["codes"], Nmax,
                          ch["finished"], ch["state"], sp["temperature"], sp["top_k"], sp["top_p"], sp["rep_penalty"],
                          cfg.stop_mel_token, advance=True)
        return st

    _SNAP = ("state", "codes", "seen", "finished")

    def _ensure_graph(self, st, sp):
        """The decode step of this workspace as a CUDA graph (captured once per workspace + sampling parameters)."""
        if st["graph"] is not None and st["graph_params"] == sp:
            return
        # warm-up once eagerly (module loading / attribute setting must not happen under capture),
        # then restore the sampler state and capture
        snap = [{k: ch[k].clone() for k in self._SNAP} for ch in st["chains"]]

        def restore():
            for ch, sn in zip(st["chains"], snap):
                for k, v in sn.items():
                    ch[k].copy_(v)
        self._decode_step(st, sp)
        torch.cuda.synchronize()
        restore()
        g = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        c0 = lib.CALLS
        with torch.cuda.stream(side):
            with torch.cuda.graph(g, stream=side):
                self._decode_step(st, sp)
        st["graph_calls"] = lib.CALLS - c0
        torch.cuda.current_stream().wait_stream(side)
        restore()
        st["graph"], st["graph_params"] = g, dict(sp)

    def _check_step_flag(self, st):
        for ch in st["chains"]:
            flag = int(ch["state"][2].item())  # TtbArState.reserved[0]: set by a timed-out wait inside the step kernel
            if flag:
                raise lib.TtbError("ar_step_kernel: internal wait timed out (code %d); results are invalid" % flag)

    @staticmethod
    def _all_finished(st):
        return all(int(ch["state"][1].item()) == 1 for ch in st["chains"])

    @staticmethod
    def _codes(st):
        cs = [ch["codes"] for ch in st["chains"]]
        return cs[0].clone() if len(cs) == 1 else torch.cat(cs, dim=0)

    @staticmethod
    def _sampling(temperature, top_k, top_p, repetition_penalty, pos_mode):
        return dict(temperature=float(temperature), top_k=int(top_k), top_p=float(top_p),
                    rep_penalty=float(repetition_penalty), pos_mode=1 if pos_mode == "ref_kv_quirk" else 0)

    def generate(self, cond_latent, text_tokens, num_candidates, max_new, uniforms=None, seed=None, temperature=0.8,
                 top_k=50, top_p=0.8, repetition_penalty=2.0, pos_mode="ref_kv_quirk", use_graph=True,
                 stop_check_every=32, trace_logits=None):
        """≙ num_candidates/bs calls of UnifiedVoice.inference_speech (autoregressive.py:535-563), all candidates in
        ONE batch with a shared-prefix KV cache. Returns int32 codes [num_candidates, max_new] padded with the
        stop token (api.py:425-426). `uniforms` [B, max_new] injects the sampling randomness (parity mode)."""
        B, Nmax = int(num_candidates), int(max_new)
        sp = self._sampling(temperature, top_k, top_p, repetition_penalty, pos_mode)
        if trace_logits is not None:
            use_graph = False
        st = self._begin(cond_latent, text_tokens, B, Nmax, uniforms, seed, sp, trace_logits)
        steps = Nmax - 1
        if steps > 0:
            if use_graph:
                self._ensure_graph(st, sp)
                done = 0
                while done < steps:
                    n = min(stop_check_every, steps - done)
                    for _ in range(n):
                        st["graph"].replay()
                    lib.add_calls(n * st["graph_calls"])
                    done += n
                    if done < steps and self._all_finished(st):
                        break
            else:
                for i in range(steps):
                    self._decode_step(st, sp)
                    if trace_logits is not None:
                        trace_logits.append(torch.cat([ch["logits"] for ch in st["chains"]], dim=0).clone())
        if st["fused"] and steps > 0:
            self._check_step_flag(st)
        return self._codes(st)

    def generate_stream(self, cond_latent, text_tokens, max_new, first_block, block, uniforms=None, seed=None,
                        temperature=0.8, top_k=50, top_p=0.8, repetition_penalty=2.0, pos_mode="ref_kv_quirk",
                        use_graph=True):
        """ONE sequence decoded block-wise: ≙ the token stream of `GPT2InferenceModel.generate_stream` /
        `sample_stream` (autoregressive.py:565-574, stream_generator.py:916-1000), which yields every sampled token
        INCLUDING the stop token and ends after it (or after `max_new` tokens). A generator of `(codes, ended)`:
        `codes` = int32 [n] all tokens so far, after the first `first_block` tokens, then every `block` tokens, and a
        last time when the stream has ended (`ended` True; the stop token, if any, is the last element)."""
        Nmax = int(max_new)
        sp = self._sampling(temperature, top_k, top_p, repetition_penalty, pos_mode)
        st = self._begin(cond_latent, text_tokens, 1, Nmax, uniforms, seed, sp)
        if use_graph and Nmax > 1:
            self._ensure_graph(st, sp)
        stop = self.cfg.stop_mel_token
        have = 1                       # tokens sampled so far (the first one comes from the prefill logits)
        target = max(1, int(first_block))
        blk = max(1, int(block))
        while True:
            want = min(target, Nmax)
            for _ in range(want - have):
                if use_graph:
                    st["graph"].replay()
                else:
                    self._decode_step(st, sp)
            if use_graph and want > have:
                lib.add_calls((want - have) * st["graph_calls"])
            have = max(have, want)
            row = st["chains"][0]["codes"][0, :have].clone()
            if st["fused"] and have > 1:
                self._check_step_flag(st)
            hit = (row == stop).nonzero()
            if hit.numel() > 0:
                yield row[: int(hit[0].item()) + 1], True
                return
            if have >= Nmax:
                yield row, True
                return
            yield row, False
            target = have + blk

    # ------------------------------------------------------------------ teacher-forced passes
    def _forward_sequences(self, emb_fn, nseq, T):
        """Runs the trunk over nseq sequences of T tokens (causal). emb_fn fills x [nseq*T, D]. Returns x."""
        D, H = self.D, self.H
        M = nseq * T
        x = torch.empty(M, D, dtype=torch.float32, device=self.dev)
        emb_fn(x)
        ws = self._alloc_trunk(M)

        def attn(qkv, o):
            lib.attention(qkv, o, nseq=nseq, T=T, H=H, ld=3 * D, ldo=D, k_off=D, v_off=2 * D, scale=0.125, causal=True)
        for lw in self.w.layers:
            self._layer(lw, x, M, ws, attn)
        return x

    def teacher_forced_logits(self, cond_latent, text_tokens, codes, pos_mode="ref_kv_quirk"):
        """Logits at every decode position when fed `codes` [B, n] (parity check of rows a1/a2)."""
        cfg, D, dev = self.cfg, self.D, self.dev
        B, n = codes.shape
        ids = self._prompt_ids(text_tokens)
        Pm = len(ids) + 1            # cond + text
        T = Pm + n + 1
        quirk = pos_mode == "ref_kv_quirk"

        def emb(x):
            xv = x.view(B, T, D)
            tid = torch.tensor(ids, dtype=torch.int32, device=dev)
            tpos = torch.arange(len(ids), dtype=torch.int32, device=dev)
            tmp = torch.empty(len(ids), D, dtype=torch.float32, device=dev)
            lib.embed(tid, tpos, len(ids), D, self.w.text_emb, self.w.text_pos, tmp)
            xv[:, 0] = cond_latent.reshape(-1).to(dev)
            xv[:, 1:Pm] = tmp
            mid = torch.cat([torch.full((B, 1), cfg.start_mel_token, dtype=torch.int32, device=dev),
                             codes.to(device=dev, dtype=torch.int32)], dim=1).contiguous()
            mpos = torch.tensor([(j + 1 if (quirk and j >= 1) else j) for j in range(n + 1)], dtype=torch.int32,
                                device=dev).repeat(B, 1).contiguous()
            tmp2 = torch.empty(B * (n + 1), D, dtype=torch.float32, device=dev)
            lib.embed(mid.view(-1), mpos.view(-1), B * (n + 1), D, self.w.mel_emb, self.w.mel_pos, tmp2)
            xv[:, Pm:] = tmp2.view(B, n + 1, D)
        x = self._forward_sequences(emb, B, T)
        M = B * T
        hn = torch.empty(M, D, dtype=torch.bfloat16, device=dev)
        lib.layernorm(x, M, D, self.w.lnf_g, self.w.lnf_b, self.w.fn_g, self.w.fn_b, out_bf16=hn)
        logits = torch.empty(M, self.V, dtype=torch.float32, device=dev)
        lib.gemm(hn, self.w.w_head, M=M, N=self.V, K=D, bias=self.w.b_head, out_f32=logits)
        return logits.view(B, T, self.V)[:, Pm:]

    def latents(self, cond_latent, text_tokens, codes):
        """≙ UnifiedVoice.forward(..., return_latent=True, clip_inputs=False) (autoregressive.py:454-512, called at
        api.py:521-524). codes [k, L] -> fp32 [k, L, D]."""
        cfg, D, dev = self.cfg, self.D, self.dev
        k, L = codes.shape
        ids = self._prompt_ids(text_tokens)
        Pm = len(ids) + 1
        T = Pm + L + 2

        def emb(x):
            xv = x.view(k, T, D)
            tid = torch.tensor(ids, dtype=torch.int32, device=dev)
            tpos = torch.arange(len(ids), dtype=torch.int32, device=dev)
            tmp = torch.empty(len(ids), D, dtype=torch.float32, device=dev)
            lib.embed(tid, tpos, len(ids), D, self.w.text_emb, self.w.text_pos, tmp)
            xv[:, 0] = cond_latent.reshape(-1).to(dev)
            xv[:, 1:Pm] = tmp
            mid = torch.cat([torch.full((k, 1), cfg.start_mel_token, dtype=torch.int32, device=dev),
                             codes.to(device=dev, dtype=torch.int32),
                             torch.full((k, 1), cfg.stop_mel_token, dtype=torch.int32, device=dev)], dim=1).contiguous()
            mpos = torch.arange(L + 2, dtype=torch.int32, device=dev).repeat(k, 1).contiguous()
            tmp2 = torch.empty(k * (L + 2), D, dtype=torch.float32, device=dev)
            lib.embed(mid.view(-1), mpos.view(-1), k * (L + 2), D, self.w.mel_emb, self.w.mel_pos, tmp2)
            xv[:, Pm:] = tmp2.view(k, L + 2, D)
        x = self._forward_sequences(emb, k, T)
        M = k * T
        out = torch.empty(M, D, dtype=torch.float32, device=dev)
        lib.layernorm(x, M, D, self.w.lnf_g, self.w.lnf_b, self.w.fn_g, self.w.fn_b, out_f32=out)
        return out.view(k, T, D)[:, Pm:Pm + L].contiguous()

    def stream_latents(self, cond_latent, text_tokens, codes):
        """The latents the streaming generator yields next to its tokens (stream_generator.py:982:
        `final_norm(hidden_states[-1][:, -1])` of the step that SAMPLED token i, i.e. of the input [start, c_0 ... c_{i-1}]
        with the KV-cache position rule of GPT2InferenceModel.forward). codes int [n] -> fp32 [n, D], one teacher-forced
        pass over the prefix instead of n cached steps (same numbers: the decode-step parity tests pin the two forms
        against each other)."""
        cfg, D, dev = self.cfg, self.D, self.dev
        codes = codes.reshape(-1)
        n = int(codes.numel())
        ids = self._prompt_ids(text_tokens)
        Pm = len(ids) + 1
        T = Pm + n

        def emb(x):
            tid = torch.tensor(ids, dtype=torch.int32, device=dev)
            tpos = torch.arange(len(ids), dtype=torch.int32, device=dev)
            lib.embed(tid, tpos, len(ids), D, self.w.text_emb, self.w.text_pos, x[1:Pm])
            x[0] = cond_latent.reshape(-1).to(dev)
            mid = torch.cat([torch.full((1,), cfg.start_mel_token, dtype=torch.int32, device=dev),
                             codes[: n - 1].to(device=dev, dtype=torch.int32)]).contiguous()
            mpos = torch.tensor([(j + 1 if j >= 1 else j) for j in range(n)], dtype=torch.int32, device=dev)
            lib.embed(mid, mpos, n, D, self.w.mel_emb, self.w.mel_pos, x[Pm:])
        x = self._forward_sequences(emb, 1, T)
        out = torch.empty(T, D, dtype=torch.float32, device=dev)
        lib.layernorm(x, T, D, self.w.lnf_g, self.w.lnf_b, self.w.fn_g, self.w.fn_b, out_f32=out)
        return out[Pm:].contiguous()
