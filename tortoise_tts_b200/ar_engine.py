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


def _rows(ch):
    """The row_start keyword of the lib calls of a chain with per-row start steps (SlotWorkspace); none otherwise."""
    return {} if ch.get("row_start") is None else {"row_start": ch["row_start"]}


def plan_batches(utterances, max_rows=lib.AR_STEP_MAX_B, max_groups=lib.AR_STEP_MAX_GROUPS, max_P=lib.AR_STEP_MAX_P):
    """Packs utterances into consecutive decode batches for AREngine.generate_grouped. `utterances`: list of
    (candidates, prompt positions P). Returns a list of batches, each a list of utterance indices in order; an utterance
    is never split. A batch holds at most `max_rows` candidates and `max_groups` utterances. An utterance with more than
    `max_rows` candidates or a prompt longer than `max_P` positions is a batch of its own (decoded by generate())."""
    batches, cur, rows = [], [], 0
    for u, (n, P) in enumerate(utterances):
        n, P = int(n), int(P)
        if n <= 0 or P <= 0:
            raise ValueError("utterance %d: %d candidates, prompt of %d positions" % (u, n, P))
        if n > max_rows or P > max_P:
            if cur:
                batches.append(cur)
            batches.append([u])
            cur, rows = [], 0
            continue
        if cur and (rows + n > max_rows or len(cur) == max_groups):
            batches.append(cur)
            cur, rows = [], 0
        cur.append(u)
        rows += n
    if cur:
        batches.append(cur)
    return batches


def clip_groups(groups, lo, hi):
    """The prompt groups [(row_begin, row_end, P, prefix), ...] of a batch as seen by the decode chain of rows [lo, hi):
    groups that overlap the chain, clipped to it, with rows counted from lo. A group that straddles two chains appears
    in both and shares its (read-only) prefix."""
    out = []
    for b, e, P, pkv in groups:
        b2, e2 = max(b, lo), min(e, hi)
        if b2 < e2:
            out.append((b2 - lo, e2 - lo, P, pkv))
    return out


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
    # How the step runs when the one-kernel form (csrc/ar_step.cu) is available: "fused" = everything in the persistent
    # kernel, whose phases grow with the batch (one CTA per SM serialises TMA wait -> MMA -> epilogue inside a phase,
    # which several small kernels per SM overlap). "mixed" = the per-op graph with its three attention kernels (prefix
    # flash + candidate stream + merge) replaced by the persistent kernel's attention phase (one launch). "auto" picks by
    # batch size: the one-kernel step for small batches only (H100 80GB HBM3, 700 W, 256 candidates, 429 steps: AR 1.73 s
    # mixed against 3.50 s fused; the batch size where the two cross, FUSED_MAX_B, has not been measured on H100).
    # "perop" = one kernel per operation: the tests' reference, and the only form for shapes the one-kernel form does not
    # cover (lib.ar_step_supported).
    MODE = _os.environ.get("TTB_AR_MODE", "auto")            # auto | fused | mixed | perop
    FUSED_MAX_B = int(_os.environ.get("TTB_AR_FUSED_MAX_B", "16"))
    # TTB_AR_CHAINS=2: in mixed mode the candidates are decoded as TWO independent half-batches on two streams inside
    # one captured step. Every kernel of the chain LN -> c_attn -> attention -> c_proj -> LN -> c_fc -> mlp.c_proj is
    # bound by its own latency except the attention (HBM-bound), so the chain of one half fills the bubbles of the
    # other; the attention then runs in compact CTAs (lib.ArStep attn_compact) that leave room for a GEMM CTA per SM.
    # measured on H100 (80GB HBM3, 700 W) at 256 candidates: AR 1839 ms with one chain, 1727 ms with two; split-K 2 / 4
    # against none: 1727 against 1795 ms; weight prefetch ahead of the dependency wait on the GEMMs that follow a
    # LayerNorm against none: 1727 / 1731 ms (inside the run-to-run spread). CHAINS_MIN_B has not been measured on H100.
    CHAINS = int(_os.environ.get("TTB_AR_CHAINS", "2"))
    CHAINS_MIN_B = int(_os.environ.get("TTB_AR_CHAINS_MIN_B", "128"))
    SPLITK_PROJ = 2      # attn.c_proj (K = D): 32 n-tiles x 2 m-tiles x 2 splits = 128 CTAs at D=1024, B=256
    SPLITK_PROJ2 = 4     # mlp.c_proj (K = 4D): 32 x 2 x 4 = 256 CTAs

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
        # a stream pool's slot (fused layout) holds prompts up to its capacity st["P"]; every other prefix is exact
        assert P == st["P"] or (st["fused"] and P <= st["P"]), (P, st["P"])
        cap = st["P"] if P != st["P"] else None
        x = st["px"][:P]
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
                    lib.ar_step_store_prefix(qkv, P, H, st["pkv"][l], **({} if cap is None else {"cap": cap}))
                else:
                    lib.ar_store_prefix(qkv, P, H, st["pk"][l], st["pv"][l])
                lib.attention(qkv, o, nseq=1, T=P, H=H, ld=3 * D, ldo=D, k_off=D, v_off=2 * D, scale=0.125, causal=True)
            self._layer(lw, x, P, ws, attn)
        lib.layernorm(x[P - 1:], 1, D, self.w.lnf_g, self.w.lnf_b, self.w.fn_g, self.w.fn_b, out_bf16=st["hn"][:1])
        lib.gemm(st["hn"], self.w.w_head, M=1, N=self.V, K=D, bias=self.w.b_head, out_f32=st["logits"])

    # ------------------------------------------------------------------ decode workspace + graph
    def _decode_state(self, B, P, Nmax, group_rows=None, group_P=None):
        """Decode workspace of B candidates. group_rows / group_P (grouped decode): the candidates of each utterance of the
        batch and its prompt length; P is then unused and every group gets its own prefix buffers (st["groups"])."""
        key = (B, P, Nmax) if group_rows is None else (B, tuple(group_rows), tuple(group_P), Nmax)
        if self._dec is not None and self._dec["key"] == key:
            return self._dec
        self._dec = None                  # release the previous workspace (KV caches) before allocating the next
        self._dec = self._build_state(key, B, P, Nmax, group_rows, group_P)
        return self._dec

    def _build_state(self, key, B, P, Nmax, group_rows=None, group_P=None, shared_prefill=False):
        """The decode workspace _decode_state describes, not kept in self._dec. shared_prefill: the groups share one set
        of prefill buffers (px, pws), which holds only while their prefills are never kept past the next one."""
        dev = self.dev
        if group_rows is None:
            ok = lib.ar_step_supported(B, self.D, self.H, P)
        else:
            ok = all(lib.ar_step_supported(B, self.D, self.H, p) for p in group_P)
            if not ok or self.MODE == "perop" or len(group_rows) > lib.AR_STEP_MAX_GROUPS:
                raise lib.TtbError("grouped decode needs the one-kernel step: %d groups (at most %d), %d rows, prompts %s "
                                   "(mode %s)" % (len(group_rows), lib.AR_STEP_MAX_GROUPS, B, list(group_P), self.MODE))
        mode = self.MODE if ok else "perop"
        if mode == "auto":
            mode = "fused" if B <= self.FUSED_MAX_B else "mixed"
        nch = self.CHAINS if (mode == "mixed" and self.CHAINS > 1 and B >= self.CHAINS_MIN_B and B % self.CHAINS == 0) else 1
        st = dict(key=key, P=P, B=B, Nmax=Nmax, mode=mode, fused=mode in ("fused", "mixed"))
        if group_rows is None:
            # ---- prompt prefill (shared by every candidate and every chain)
            self._prefix_state(st, P)
        else:
            st["groups"] = []
            b = 0
            for n, p in zip(group_rows, group_P):
                gs = dict(P=p, fused=True, b0=b, b1=b + n)
                if shared_prefill and st["groups"]:
                    gs["px"], gs["pws"] = st["groups"][0]["px"], st["groups"][0]["pws"]
                self._prefix_state(gs, p)
                st["groups"].append(gs)
                b += n
        # ---- decode workspaces: one per chain (contiguous candidate ranges)
        per = B // nch
        st["chains"] = [self._chain_state(st, per, c * per, compact=nch > 1) for c in range(nch)]
        # the per-row sampling settings (include/ttb.h TtbSampleParams, 8 words a row) read by a per-row decode
        st["params"] = torch.zeros(B, 8, dtype=torch.int32, device=dev)
        for ch in st["chains"]:
            ch["params"] = st["params"][ch["b0"]: ch["b0"] + ch["B"]]
        st["sides"] = [torch.cuda.Stream(device=dev) for _ in range(nch - 1)] if dev.type == "cuda" else []
        st["graph"] = None
        st["graph_params"] = None
        return st

    def _prefix_state(self, st, P):
        """Prefill buffers and the prompt-prefix KV cache of one prompt of P positions, into the dict `st`."""
        cfg, D, dev = self.cfg, self.D, self.dev
        L, H = cfg.ar_layers, self.H
        if "px" not in st:
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

    def _chain_state(self, st, B, b0, compact=False):
        """Decode workspace of candidates [b0, b0 + B): residual stream, trunk buffers, candidate KV cache, sampler state."""
        cfg, D, H, dev = self.cfg, self.D, self.H, self.dev
        L, Nmax = cfg.ar_layers, st["Nmax"]
        ch = dict(B=B, b0=b0, P=st["P"], Nmax=Nmax, mode=st["mode"], fused=st["fused"], compact=compact)
        if "groups" in st:
            ch["groups"] = clip_groups([(g["b0"], g["b1"], g["P"], g["pkv"]) for g in st["groups"]], b0, b0 + B)
            ch["P"] = max(g[2] for g in ch["groups"])
            ch["pkv"] = ch["groups"][0][3]
            ch["ckv"] = torch.zeros(L, B, H, Nmax, 2, 64, dtype=torch.bfloat16, device=dev)
        elif st["fused"]:
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
                            attn_compact=bool(st.get("compact")), groups=st.get("groups"), **_rows(st))
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
            self._sample(sp, st["logits"], self.V, st)
            if sp.get("capture"):
                self._capture(st)
            return
        hd = self._step_handle(st, sp["pos_mode"]) if st["mode"] == "mixed" else None
        lib.ar_embed_step(st["codes"], Nmax, st["state"], self.w.mel_emb, self.w.mel_pos, B, D, sp["pos_mode"], x,
                          **_rows(st))
        # Skinny-M decode (M = B candidates): every GEMM is weight-streaming bound, so the grid is widened with
        # 32-column tiles and, for the two GEMMs that feed the residual stream, split-K; their partial sums, bias and
        # the residual add are folded into the LayerNorm that follows (fixed summation order -> deterministic).
        # c_attn, c_fc and mel_head follow a LayerNorm, which triggers its dependents early: they fetch their weights
        # ahead of griddepcontrol.wait (w_static).
        kb = D // 64
        s1 = min(self.SPLITK_PROJ, kb)
        s2 = min(self.SPLITK_PROJ2, 4 * kb)
        pa, pb = st["part_a"], st["part_b"]
        prev = None   # (partials, nsplit, bias) of the previous layer's mlp.c_proj, folded into the next LayerNorm
        for l, lw in enumerate(self.w.layers):
            if prev is None:
                lib.layernorm(x, B, D, lw["ln1_g"], lw["ln1_b"], out_bf16=ws["a"])
            else:
                lib.residual_layernorm(x, B, D, prev[0], prev[1], B * D, prev[2], lw["ln1_g"], lw["ln1_b"], out_bf16=ws["a"])
            lib.gemm(ws["a"], lw["wqkv"], M=B, N=3 * D, K=D, bias=lw["bqkv"], out_bf16=ws["qkv"], tile_n=32, w_static=True)
            if hd is not None:
                hd.step(phase_mask=4, layer_begin=l, layer_end=l + 1)     # attention phase of the persistent kernel
            else:
                lib.ar_decode_attention(ws["qkv"], st["pk"][l], st["pv"][l], st["ck"][l], st["cv"][l], st["state"], B, H,
                                        P, Nmax, ws["o"], st["att_o"], st["att_lse"])
            lib.gemm(ws["o"], lw["wproj"], M=B, N=D, K=D, out_f32=pa, outf_bstride=B * D, tile_n=32, splitk=max(s1, 2))
            lib.residual_layernorm(x, B, D, pa, self._nsplit(kb, max(s1, 2)), B * D, lw["bproj"], lw["ln2_g"], lw["ln2_b"],
                                   out_bf16=ws["a"])
            lib.gemm(ws["a"], lw["wfc"], M=B, N=4 * D, K=D, bias=lw["bfc"], act=lib.ACT_GELU_NEW, out_bf16=ws["h"],
                     tile_n=32, w_static=True)
            lib.gemm(ws["h"], lw["wproj2"], M=B, N=D, K=4 * D, out_f32=pb, outf_bstride=B * D, tile_n=32, splitk=max(s2, 2))
            prev = (pb, self._nsplit(4 * kb, max(s2, 2)), lw["bproj2"])
        lib.residual_layernorm(x, B, D, prev[0], prev[1], B * D, prev[2], self.w.lnf_g, self.w.lnf_b, self.w.fn_g,
                               self.w.fn_b, out_bf16=st["hn"])
        lib.gemm(st["hn"], self.w.w_head, M=B, N=self.V, K=D, bias=self.w.b_head, out_f32=st["logits"], w_static=True)
        self._sample(sp, st["logits"], self.V, st)
        if sp.get("capture"):
            self._capture(st)

    def _capture(self, ch):
        """Latent capture of one chain, after its sampler: row b's latent of the token just sampled goes to
        ch["lat"][b, step - 1] (the rows of the batch's [B, Nmax, D] buffer that belong to this chain)."""
        w = self.w
        lib.ar_capture_latents(ch["x"], ch["B"], self.D, w.lnf_g, w.lnf_b, w.fn_g, w.fn_b, ch["state"], ch["Nmax"],
                               ch["lat"], ch["Nmax"] * self.D, **_rows(ch))

    def _sample(self, sp, logits, ld_logits, ch):
        """The sampler over the logits of one chain (ld_logits = 0: row 0 for every candidate); the typical-set entry
        when `sp` turns the filter on, the per-row entry (each row's settings from ch["params"]) when `sp` is per-row."""
        Nmax = ch["Nmax"]
        if sp.get("per_row"):
            lib.ar_sample_params(logits, ld_logits, self.V, ch["B"], ch["uniforms"], Nmax, ch["seen"], ch["codes"], Nmax,
                                 ch["finished"], ch["state"], ch["params"], self.cfg.stop_mel_token, advance=True,
                                 **_rows(ch))
            return
        args = (logits, ld_logits, self.V, ch["B"], ch["uniforms"], Nmax, ch["seen"], ch["codes"], Nmax, ch["finished"],
                ch["state"], sp["temperature"], sp["top_k"], sp["top_p"], sp["rep_penalty"], self.cfg.stop_mel_token)
        if sp.get("typical_mass") is None:
            lib.ar_sample(*args, advance=True, **_rows(ch))
        else:
            assert ch.get("row_start") is None, "the typical sampler has no per-row start steps"
            lib.ar_sample_typical(*args, sp["typical_mass"], advance=True)

    def _begin(self, cond_latent, text_tokens, B, Nmax, uniforms, seed, sp, trace_logits=None, prefill_events=None):
        """Workspace reset + prompt prefill + the first sampled token of every candidate. `prefill_events`: None or a
        pair of CUDA events recorded around the prefill."""
        cfg, dev = self.cfg, self.dev
        P = len(text_tokens) + 4  # cond + [start, tokens(padded), stop] + start_mel
        st = self._decode_state(B, P, Nmax)
        if uniforms is None:
            g = torch.Generator(device=dev)
            g.manual_seed(0 if seed is None else int(seed))
            uniforms = torch.rand(B, Nmax, generator=g, device=dev)
        uniforms = uniforms.to(device=dev, dtype=torch.float32)
        if prefill_events is not None:
            prefill_events[0].record()
        self._prefill(cond_latent, text_tokens, st)
        if prefill_events is not None:
            prefill_events[1].record()
        if trace_logits is not None:   # parity hook (eager mode): logits the sampler sees at every step
            trace_logits.append(st["logits"][:1].expand(B, -1).clone())
        for ch in st["chains"]:
            self._reset_chain(ch, uniforms)
            self._sample(sp, st["logits"], 0, ch)
        return st

    def _reset_chain(self, ch, uniforms):
        """Sampler state of one chain before the first token; `uniforms` [B, Nmax] of the whole batch."""
        ch["state"].zero_()
        self._reset_rows(ch, slice(0, ch["B"]), uniforms[ch["b0"]: ch["b0"] + ch["B"]])

    def _reset_rows(self, ch, rows, uniforms):
        """Sampler state of rows `rows` (a slice) of one chain before their first token: uniforms [rows, Nmax], seen
        bits {1, start_mel}, not finished, codes filled with the stop token."""
        cfg = self.cfg
        w, bit = divmod(cfg.start_mel_token, 32)
        ch["uniforms"][rows].copy_(uniforms)
        ch["finished"][rows] = 0
        ch["codes"][rows] = cfg.stop_mel_token
        ch["seen"][rows] = 0
        # HF's repetition penalty sees the fake prompt ids {1, start_mel} (autoregressive.py:546-548)
        ch["seen"][rows, 0] = 2
        ch["seen"][rows, w] |= (1 << bit) if bit < 31 else -(1 << 31)

    def _begin_grouped(self, cond_latent, text_tokens_list, counts, Nmax, uniforms_list, seed, sp, trace_logits=None,
                       prefill_events=None, params=None):
        """_begin for a batch of utterances: one prefill per utterance into its own prefix, and the first token of every
        row sampled from its utterance's prefill logits (one sampler call per chain, so the step counter advances once).
        `cond_latent`: one conditioning latent for every utterance, or a list with one per utterance.
        `prefill_events`: None or a pair of CUDA events recorded around the prefills. `params`: the per-row settings
        table (lib.sample_params_table, one row per decode row) of a per-row `sp`, written before the first token."""
        dev = self.dev
        conds = list(cond_latent) if isinstance(cond_latent, (list, tuple)) else [cond_latent] * len(counts)
        if len(conds) != len(counts):
            raise ValueError("%d conditioning latents for %d utterances" % (len(conds), len(counts)))
        Ps = [len(t) + 4 for t in text_tokens_list]
        st = self._decode_state(sum(counts), None, Nmax, counts, Ps)
        us = []
        for n, u in zip(counts, uniforms_list if uniforms_list is not None else [None] * len(counts)):
            if u is None:          # as generate(): every utterance draws its own table from the same seed
                g = torch.Generator(device=dev)
                g.manual_seed(0 if seed is None else int(seed))
                u = torch.rand(n, Nmax, generator=g, device=dev)
            us.append(u.to(device=dev, dtype=torch.float32))
        uniforms = torch.cat(us, dim=0)
        if params is not None:
            st["params"].copy_(params)
        if prefill_events is not None:
            prefill_events[0].record()
        for gs, cond, toks in zip(st["groups"], conds, text_tokens_list):
            self._prefill(cond, toks, gs)
        if prefill_events is not None:
            prefill_events[1].record()
        first = torch.cat([gs["logits"].expand(gs["b1"] - gs["b0"], -1) for gs in st["groups"]], dim=0)
        if trace_logits is not None:
            trace_logits.append(first.clone())
        for ch in st["chains"]:
            self._reset_chain(ch, uniforms)
            ch["logits"].copy_(first[ch["b0"]: ch["b0"] + ch["B"]])
            self._sample(sp, ch["logits"], self.V, ch)
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
    def _sampling(temperature, top_k, top_p, repetition_penalty, pos_mode, typical_mass=None, capture=False,
                  per_row=False):
        """The sampling parameters of a decode; also the key of the captured step graph, so a change of any of them
        (the typical mass and the latent capture included) captures a new graph. typical_mass None = no typical filter.
        capture: every step ends with ttb_ar_capture_latents into each chain's ch["lat"]; without it the step (and its
        graph) is what it is without this option. per_row: the sampler reads every row's settings from the decode
        state's table st["params"] (ttb_ar_sample_params), which is not part of the key: new settings in the table reuse
        the graph, and the scalar settings here are unused."""
        sp = dict(temperature=float(temperature), top_k=int(top_k), top_p=float(top_p),
                  rep_penalty=float(repetition_penalty), pos_mode=1 if pos_mode == "ref_kv_quirk" else 0)
        if capture:
            sp["capture"] = True
        if per_row:
            sp["per_row"] = True
        if typical_mass is not None:
            m = float(typical_mass)
            if not 0.0 < m <= 1.0:
                raise ValueError("typical_mass must lie in (0, 1], got %r" % (typical_mass,))
            sp["typical_mass"] = m
        return sp

    def generate(self, cond_latent, text_tokens, num_candidates, max_new, uniforms=None, seed=None, temperature=0.8,
                 top_k=50, top_p=0.8, repetition_penalty=2.0, pos_mode="ref_kv_quirk", use_graph=True,
                 stop_check_every=32, trace_logits=None, typical_mass=None, prefill_events=None):
        """≙ num_candidates/bs calls of UnifiedVoice.inference_speech (autoregressive.py:535-563), all candidates in
        ONE batch with a shared-prefix KV cache. Returns int32 codes [num_candidates, max_new] padded with the
        stop token (api.py:425-426). `uniforms` [B, max_new] injects the sampling randomness (parity mode).
        `typical_mass` (in (0, 1]) turns on the reference's typical-set filter (TypicalLogitsWarper after the repetition
        penalty, autoregressive.py:558); None leaves it off. `prefill_events`: None or a pair of CUDA events recorded
        around the prompt prefill."""
        B, Nmax = int(num_candidates), int(max_new)
        sp = self._sampling(temperature, top_k, top_p, repetition_penalty, pos_mode, typical_mass)
        if trace_logits is not None:
            use_graph = False
        st = self._begin(cond_latent, text_tokens, B, Nmax, uniforms, seed, sp, trace_logits, prefill_events)
        self._decode(st, sp, Nmax - 1, use_graph, stop_check_every, trace_logits)
        return self._codes(st)

    def generate_grouped(self, cond_latent, text_tokens_list, counts, max_new, uniforms_list=None, seed=None,
                         temperature=0.8, top_k=50, top_p=0.8, repetition_penalty=2.0, pos_mode="ref_kv_quirk",
                         use_graph=True, stop_check_every=32, trace_logits=None, typical_mass=None,
                         prefill_events=None, row_settings=None):
        """Several utterances decoded in ONE batch: utterance u contributes counts[u] candidates that attend to its own
        prompt (text_tokens_list[u]; `cond_latent` is one conditioning latent for all, or a list with one per utterance,
        each utterance's latent then starting its own prompt). Returns one int32 codes tensor [counts[u], max_new]
        per utterance, each as generate(cond_latent, text_tokens_list[u], counts[u], max_new, uniforms_list[u], ...)
        returns it. At most lib.AR_STEP_MAX_GROUPS utterances, lib.AR_STEP_MAX_B rows and prompts of
        lib.AR_STEP_MAX_P positions (plan_batches packs within these limits); the one-kernel step is required.
        `prefill_events`: None or a pair of CUDA events recorded around the prefills. `row_settings`: None, or one dict
        per utterance of sampling settings (keys temperature, top_k, top_p, repetition_penalty, typical_mass; a missing
        key takes the argument of this call) for all of its rows: utterance u then samples as generate(...) with its
        settings, through the per-row sampler."""
        counts = [int(n) for n in counts]
        if len(counts) != len(text_tokens_list) or (uniforms_list is not None and len(uniforms_list) != len(counts)):
            raise ValueError("one entry of counts (and of uniforms_list) per utterance")
        Nmax = int(max_new)
        params = self._row_params(row_settings, counts, temperature, top_k, top_p, repetition_penalty, typical_mass)
        sp = self._sampling(temperature, top_k, top_p, repetition_penalty, pos_mode,
                            typical_mass if params is None else None, per_row=params is not None)
        if trace_logits is not None:
            use_graph = False
        st = self._begin_grouped(cond_latent, text_tokens_list, counts, Nmax, uniforms_list, seed, sp, trace_logits,
                                 prefill_events, params)
        self._decode(st, sp, Nmax - 1, use_graph, stop_check_every, trace_logits)
        codes = self._codes(st)
        return [codes[g["b0"]: g["b1"]].clone() for g in st["groups"]]

    def _row_params(self, row_settings, counts, temperature, top_k, top_p, repetition_penalty, typical_mass):
        """The per-row settings table of a grouped decode (lib.sample_params_table, validated) from one settings dict
        per group, each expanded to its group's rows over the call's own settings; None without row_settings."""
        if row_settings is None:
            return None
        if len(row_settings) != len(counts):
            raise ValueError("%d row_settings for %d utterances" % (len(row_settings), len(counts)))
        base = dict(temperature=temperature, top_k=top_k, top_p=top_p, repetition_penalty=repetition_penalty,
                    typical_mass=typical_mass)
        rows = []
        for n, rs in zip(counts, row_settings):
            unknown = set(rs) - set(base)
            if unknown:
                raise TypeError("unknown sampling settings: %s" % sorted(unknown))
            rows += [{**base, **rs}] * n
        return lib.sample_params_table(rows, self.dev)

    def _decode(self, st, sp, steps, use_graph, stop_check_every, trace_logits):
        """The decode loop after the first token: `steps` steps (graph replays polled for the stop every
        stop_check_every steps, or eager with the logits traced)."""
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

    def generate_stream(self, cond_latent, text_tokens, max_new, first_block, block, uniforms=None, seed=None,
                        temperature=0.8, top_k=50, top_p=0.8, repetition_penalty=2.0, pos_mode="ref_kv_quirk",
                        use_graph=True, typical_mass=None):
        """ONE sequence decoded block-wise: ≙ the token stream of `GPT2InferenceModel.generate_stream` /
        `sample_stream` (autoregressive.py:565-574, stream_generator.py:916-1000), which yields every sampled token
        INCLUDING the stop token and ends after it (or after `max_new` tokens). A generator of `(codes, ended)`:
        `codes` = int32 [n] all tokens so far, after the first `first_block` tokens, then every `block` tokens, and a
        last time when the stream has ended (`ended` True; the stop token, if any, is the last element)."""
        Nmax = int(max_new)
        sp = self._sampling(temperature, top_k, top_p, repetition_penalty, pos_mode, typical_mass)
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

    def generate_grouped_stream(self, cond_latent, text_tokens_list, max_new, first_block, block, uniforms_list=None,
                                seed=None, temperature=0.8, top_k=50, top_p=0.8, repetition_penalty=2.0,
                                pos_mode="ref_kv_quirk", use_graph=True, typical_mass=None, row_settings=None):
        """generate_stream for several utterances, ONE row each, decoded in one grouped batch (limits of
        generate_grouped); each row attends to its own prompt text_tokens_list[u], after its own conditioning latent
        (`cond_latent`: one for all, or a list). `max_new`: the cap of every row, or a list with one per row; the batch
        decodes up to the largest. uniforms_list[u]: [1, >= max_new[u]] (padded here to the batch width).
        Every step also captures the latents the streaming generator yields next to its tokens (ttb_ar_capture_latents;
        latent 0 is the prefill's last row), so no teacher-forced pass is needed to decode them.
        A generator of `(codes, ended, latents)`, after the first `first_block` tokens, then every `block` tokens, until
        every row has ended: codes[u] = int32 [n_u] the tokens of row u so far, ended[u] as generate_stream decides it
        for that row alone (its stop token, kept as the last element, or its cap reached); a row that has ended keeps
        its last codes in later yields. `latents` fp32 [rows, max(max_new), D]: latents[u, i] belongs to codes[u][i];
        the buffer belongs to the decode workspace and stays valid until the next decode. `row_settings`: one
        sampling-settings dict per row, as for generate_grouped."""
        n = len(text_tokens_list)
        caps = [int(m) for m in max_new] if isinstance(max_new, (list, tuple)) else [int(max_new)] * n
        if len(caps) != n or min(caps) < 1:
            raise ValueError("one cap >= 1 per row: %s for %d rows" % (caps, n))
        Nmax, D = max(caps), self.D
        us = None
        if uniforms_list is not None:
            if len(uniforms_list) != n:
                raise ValueError("one uniforms table per row")
            us = []
            for u, c in zip(uniforms_list, caps):
                u = u.to(device=self.dev, dtype=torch.float32).reshape(1, -1)
                if u.shape[1] < c:
                    raise ValueError("uniforms of %d steps for a cap of %d" % (u.shape[1], c))
                us.append(torch.nn.functional.pad(u[:, :Nmax], (0, max(0, Nmax - u.shape[1]))))
        params = self._row_params(row_settings, [1] * n, temperature, top_k, top_p, repetition_penalty, typical_mass)
        sp = self._sampling(temperature, top_k, top_p, repetition_penalty, pos_mode,
                            typical_mass if params is None else None, capture=True, per_row=params is not None)
        st = self._begin_grouped(cond_latent, text_tokens_list, [1] * n, Nmax, us, seed, sp, params=params)
        if "lat" not in st:
            st["lat"] = torch.empty(n, Nmax, D, dtype=torch.float32, device=self.dev)
        lat = st["lat"]
        for ch in st["chains"]:
            ch["lat"] = lat[ch["b0"]: ch["b0"] + ch["B"]]
        w = self.w
        for gs in st["groups"]:          # latent 0: final norms of the prefill's last row (the start mel token)
            lib.layernorm(gs["px"][gs["P"] - 1:], 1, D, w.lnf_g, w.lnf_b, w.fn_g, w.fn_b, out_f32=lat[gs["b0"], 0])
        if use_graph and Nmax > 1:
            self._ensure_graph(st, sp)
        stop = self.cfg.stop_mel_token
        have = 1
        target = max(1, int(first_block))
        blk = max(1, int(block))
        ended, out = [False] * n, [None] * n
        while True:
            # a row's blocks end where generate_stream would end them: at its own cap
            want = min(target, max(c for c, e in zip(caps, ended) if not e))
            for _ in range(want - have):
                if use_graph:
                    st["graph"].replay()
                else:
                    self._decode_step(st, sp)
            if use_graph and want > have:
                lib.add_calls((want - have) * st["graph_calls"])
            have = max(have, want)
            codes = self._codes(st)[:, :have]
            if st["fused"] and have > 1:
                self._check_step_flag(st)
            host = codes.cpu()
            for u in range(n):
                if ended[u]:
                    continue
                m = min(have, caps[u])
                hit = (host[u, :m] == stop).nonzero()
                if hit.numel() > 0:
                    out[u], ended[u] = codes[u, : int(hit[0].item()) + 1], True
                else:
                    out[u], ended[u] = codes[u, :m], m >= caps[u]
            yield list(out), list(ended), lat
            if all(ended):
                return
            target = have + blk

    def slot_workspace(self, capacity, max_new, temperature=0.8, top_k=50, top_p=0.8, repetition_penalty=2.0,
                       pos_mode="ref_kv_quirk", use_graph=True):
        """A decode workspace of `capacity` one-row slots that rows join and leave while it runs (SlotWorkspace). The
        sampling settings are the default of every row; SlotWorkspace.admit may give a row its own."""
        defaults = dict(temperature=temperature, top_k=top_k, top_p=top_p, repetition_penalty=repetition_penalty)
        return SlotWorkspace(self, capacity, max_new, self._sampling(temperature, top_k, top_p, repetition_penalty,
                                                                     pos_mode, capture=True), use_graph, defaults)

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


class SlotWorkspace:
    """Continuous batching: a grouped decode of `capacity` one-row groups (slots) whose step graph is captured once, and
    into which a row joins whenever a slot is free. Every slot has a prompt prefix of lib.AR_STEP_MAX_P positions
    (include/ttb.h ttb_ar_step_store_prefix_cap) and its own start step (TtbArStepArgs.row_start): a row admitted when
    the shared step counter reads s has row_start s - 1, so it samples exactly the tokens that a decode of its own from
    step 0 samples. Every step captures the latents (ttb_ar_capture_latents_rows). The step forms are those of the
    grouped decode (fused up to FUSED_MAX_B rows, mixed, two chains from CHAINS_MIN_B rows); the per-op form has no
    groups and raises. A row may sample with its own settings: `admit` writes them into the slot's entry of the
    settings table (st["params"]). While every row has the workspace's settings, the step samples with the scalar
    sampler, as a workspace without per-row settings does. The first row admitted with other settings switches the
    workspace to the per-row sampler (ttb_ar_sample_params, one new step graph, captured then); from there on rows with
    any settings join without another capture. All calls enqueue on the current CUDA stream."""

    def __init__(self, eng, capacity, max_new, sp, use_graph=True, defaults=None):
        capacity, Nmax = int(capacity), int(max_new)
        if not 1 <= capacity <= lib.AR_STEP_MAX_GROUPS:
            raise ValueError("a slot workspace has 1..%d slots, got %d" % (lib.AR_STEP_MAX_GROUPS, capacity))
        Pcap = lib.AR_STEP_MAX_P
        if eng.MODE == "perop" or not lib.ar_step_supported(capacity, eng.D, eng.H, Pcap):
            raise lib.TtbError("a slot workspace needs the one-kernel step (mode %s)" % eng.MODE)
        self.eng, self.sp, self.capacity, self.Nmax, self.P_cap = eng, sp, capacity, Nmax, Pcap
        self.defaults = dict(defaults or {})
        self._default_words = lib.sample_params_row(**self.defaults)
        self.use_graph = use_graph and eng.dev.type == "cuda"
        dev, D = eng.dev, eng.D
        st = eng._build_state(("slots", capacity, Nmax), capacity, None, Nmax, [1] * capacity, [Pcap] * capacity,
                              shared_prefill=True)
        for gs in st["groups"]:
            # positions past a slot's prompt are loaded with its last chunk and weighted by 0: they must be finite
            gs["pkv"].zero_()
        st["row_start"] = torch.zeros(capacity, dtype=torch.int32, device=dev)
        st["lat"] = torch.zeros(capacity, Nmax, D, dtype=torch.float32, device=dev)
        st["params"].copy_(torch.tensor(self._default_words, dtype=torch.int32).expand(capacity, -1))
        self.where = []                       # slot -> (chain, row in the chain)
        for ch in st["chains"]:
            ch["row_start"] = st["row_start"][ch["b0"]: ch["b0"] + ch["B"]]
            ch["lat"] = st["lat"][ch["b0"]: ch["b0"] + ch["B"]]
            eng._reset_chain(ch, torch.zeros(capacity, Nmax, device=dev))
            ch["finished"].fill_(1)           # an idle slot samples nothing
            self.where += [(ch, r) for r in range(ch["B"])]
        self.st = st
        self.step = 0                         # host copy of every chain's state.step
        self.rs = torch.zeros(capacity, dtype=torch.int32)      # host copy of row_start
        self.live = [False] * capacity
        self._first_state = torch.zeros(64, dtype=torch.int32, device=dev)   # scratch counter of the first token
        for ch in st["chains"]:
            eng._step_handle(ch, sp["pos_mode"])
        if self.use_graph:
            eng._ensure_graph(st, sp)

    def admit(self, slot, cond_latent, text_tokens, uniforms_row, settings=None):
        """Starts a row in the free slot `slot`: its sampling settings in the slot's entry of the settings table,
        prompt prefill into the slot's prefix, the slot's P in the step's group table, its sampler state (as
        _reset_chain), latent 0, its row_start, and its first token, sampled from the prefill logits with the slot's
        settings and a scratch counter at 0 (the shared counter does not move). uniforms_row: [n] with n <= max_new.
        `settings`: a dict of temperature / top_k / top_p / repetition_penalty over the workspace's defaults (ValueError
        for a bad value, before anything is enqueued); settings other than the defaults switch the workspace to the
        per-row sampler if it is not there yet. Returns the prompt length P."""
        eng, sp = self.eng, self.sp
        if self.live[slot]:
            raise ValueError("slot %d is in use" % slot)
        P = len(text_tokens) + 4
        if P > self.P_cap:
            raise ValueError("a prompt of %d positions (a slot holds %d)" % (P, self.P_cap))
        unknown = set(settings or {}) - set(self.defaults)
        if unknown:
            raise TypeError("unknown sampling settings: %s" % sorted(unknown))
        words = lib.sample_params_row(**{**self.defaults, **(settings or {})})
        if words != self._default_words and not self.sp.get("per_row"):
            self._use_per_row()
            sp = self.sp
        ch, r = self.where[slot]
        ch["params"][r].copy_(torch.tensor(words, dtype=torch.int32))
        gs = self.st["groups"][slot]
        eng._prefill(cond_latent, text_tokens, gs)
        eng._step_handle(ch, sp["pos_mode"]).set_group_len(r, P)
        u = torch.zeros(1, self.Nmax, dtype=torch.float32, device=eng.dev)
        n = min(int(uniforms_row.numel()), self.Nmax)
        u[0, :n] = uniforms_row.reshape(-1)[:n].to(device=eng.dev, dtype=torch.float32)
        eng._reset_rows(ch, slice(r, r + 1), u)
        w = eng.w
        lib.layernorm(gs["px"][P - 1:], 1, eng.D, w.lnf_g, w.lnf_b, w.fn_g, w.fn_b, out_f32=ch["lat"][r, 0])
        self.rs[slot] = self.step - 1
        self._first_state.zero_()
        Nmax = self.Nmax
        args = (gs["logits"], eng.V, eng.V, 1, ch["uniforms"][r:r + 1], Nmax, ch["seen"][r:r + 1], ch["codes"][r:r + 1],
                Nmax, ch["finished"][r:r + 1], self._first_state)
        if sp.get("per_row"):
            lib.ar_sample_params(*args, ch["params"][r:r + 1], eng.cfg.stop_mel_token, advance=False)
        else:
            lib.ar_sample(*args, sp["temperature"], sp["top_k"], sp["top_p"], sp["rep_penalty"], eng.cfg.stop_mel_token,
                          advance=False)
        self.live[slot] = True
        return P

    def _use_per_row(self):
        """Switches the step to the per-row sampler (every row's entry of st["params"] already holds its settings) and
        captures its graph; called between steps, on a free slot's admission."""
        self.sp = dict(self.sp, per_row=True)
        if self.use_graph:
            self.eng._ensure_graph(self.st, self.sp)

    def release(self, slot):
        """Frees a slot: its row stops sampling, and from the next advance on it is re-based every time so that it
        attends to a few positions only (the kernels clamp it anyway)."""
        ch, r = self.where[slot]
        ch["finished"][r] = 1
        self.live[slot] = False

    def tokens(self, slot):
        """Tokens sampled so far by the row in `slot`."""
        return self.step - int(self.rs[slot])

    def advance(self, n):
        """n decode steps of every slot (graph replays)."""
        eng, st = self.eng, self.st
        for s in range(self.capacity):
            if not self.live[s]:
                self.rs[s] = self.step - 1
        st["row_start"].copy_(self.rs)
        for _ in range(int(n)):
            if self.use_graph:
                st["graph"].replay()
            else:
                eng._decode_step(st, self.sp)
        if self.use_graph:
            lib.add_calls(int(n) * st["graph_calls"])
        self.step += int(n)

    def check(self):
        """Raises if a step reported a timed-out internal wait (fused step)."""
        if self.st["fused"]:
            self.eng._check_step_flag(self.st)

    def codes(self):
        """int32 [capacity, max_new]: row s holds the tokens of slot s at columns [0, tokens(s))."""
        return self.eng._codes(self.st)

    @property
    def latents(self):
        """fp32 [capacity, max_new, D]: latents[s, i] belongs to token i of slot s."""
        return self.st["lat"]
