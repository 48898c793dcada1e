"""GPU: the per-row start steps of the stream pool (TtbArStepArgs.row_start and the _rows entry points) against plain
float64 restatements of each operation, with every row at its own step j_b = state.step - row_start[b].

The rows of one launch are given very different j_b: 1 (only the new token), the 16-position chunk and ring seams (2, 16,
17, 32, 33), Nmax - 1 and Nmax, and both clamp directions of include/ttb.h (row_start 1000 steps back, and row_start
ahead of the step). Whatever a row must not read is poisoned with large finite values (a correct kernel may load a
masked tile and weight it by 0, so no NaN or inf there), and whatever it must not write holds canaries inside the
allocation: a wrong index changes a checked value instead of addressing memory outside the buffers. Each family also
checks, on the reference side, that the mutant it guards against (an attended stale position, the neighbouring uniform
column, a latent one column off) would fail its bound."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gpu_util import report
from test_gpu_decode_perop import START, STOP, _hf_sample, _seen_mask
from test_gpu_decode_perop import V as V_SAMPLER

pytestmark = pytest.mark.gpu

PH_ATTN = 4
H, L, NMAX, PCAP = 16, 2, 430, 352          # PCAP: a slot's prefix capacity (lib.AR_STEP_MAX_P)
D = H * 64
STEP = 600                                   # the shared counter state.step of the attention launches
ABOVE, BELOW = "above", "below"
J_CLASSES = [NMAX, 1, NMAX - 1, 2, ABOVE, 16, 33, BELOW, 32, 17]    # neighbours differ sharply
PROMPTS = [1, 13, 17, 174, 351, 352]
ATTN_BOUND = 8e-3                            # test_step_attention_phase: bf16 softmax weights in P V
POISON_V = 1e4

LAYOUTS = {
    # one group per row, as the slot workspace lays out its slots
    "slots7": [1] * 7, "slots32": [1] * 32, "slots128": [1] * 128, "slots256": [1] * 256,
    # groups of many rows: a unit holds more rows than a CTA has warps, so the next row's KV stream is started
    # (with that row's own chunk count) while the current one is finished
    "shared128": [100, 28], "shared256": [180, 76],
}
KERNELS = {  # attention-only launches (one layer) and the cooperative step over two layers (include/ttb.h)
    "attn_only": (False, 1, 2), "attn_compact": (True, 1, 2), "cooperative": (False, 0, 2)}


def _row_starts(n, shift, step, classes):
    rs = []
    for b in range(n):
        c = classes[(b + shift) % len(classes)]
        rs.append(step - 1000 if c == ABOVE else step + 3 if c == BELOW else step - c)
    return torch.tensor(rs, dtype=torch.int32)


def _team(value):
    """Sets TTB_AR_STEP_TEAM (None = the planner's default) and returns a function that restores the environment."""
    saved = os.environ.get("TTB_AR_STEP_TEAM")
    if value is None:
        os.environ.pop("TTB_AR_STEP_TEAM", None)
    else:
        os.environ["TTB_AR_STEP_TEAM"] = str(value)

    def restore():
        if saved is None:
            os.environ.pop("TTB_AR_STEP_TEAM", None)
        else:
            os.environ["TTB_AR_STEP_TEAM"] = saved
    return restore


def _pool_step(sizes, compact, seed):
    """A stand-alone ArStep with row_start whose groups have prefixes of PCAP positions (set_group_len picks their P).
    cand_kv is a view into an allocation with a guard row in front and a guard layer + row behind."""
    from tortoise_tts_b200 import lib
    dev = "cuda"
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    B, G, V = sum(sizes), len(sizes), 300

    def rn(*s, scale=1.0):
        return torch.randn(*s, generator=g, device=dev) * scale
    layers = [dict(ln1_g=1 + rn(D, scale=0.1), ln1_b=rn(D, scale=0.1), ln2_g=1 + rn(D, scale=0.1), ln2_b=rn(D, scale=0.1),
                   wqkv=rn(3 * D, D, scale=0.03).to(torch.bfloat16), bqkv=rn(3 * D, scale=0.1),
                   wproj=rn(D, D, scale=0.03).to(torch.bfloat16), bproj=rn(D, scale=0.1),
                   wfc=rn(4 * D, D, scale=0.03).to(torch.bfloat16), bfc=rn(4 * D, scale=0.1),
                   wproj2=rn(D, 4 * D, scale=0.02).to(torch.bfloat16), bproj2=rn(D, scale=0.1)) for _ in range(L)]
    row = H * NMAX * 128
    flat = torch.empty((L + 1) * (B + 1) * row, dtype=torch.bfloat16, device=dev).normal_(generator=g)
    cand = flat[row: row + L * B * row].view(L, B, H, NMAX, 2, 64)
    pfx = torch.zeros(G, L, H, PCAP, 2, 64, dtype=torch.bfloat16, device=dev)
    groups, gidx, b = [], [], 0
    for i, n in enumerate(sizes):
        groups.append((b, b + n, PCAP, pfx[i]))
        gidx += [i] * n
        b += n
    rs = torch.zeros(B, dtype=torch.int32, device=dev)
    t = dict(layers=layers, w_head=rn(V, D, scale=0.03).to(torch.bfloat16), b_head=rn(V, scale=0.1),
             lnf_g=1 + rn(D, scale=0.1), lnf_b=rn(D, scale=0.1), fn_g=1 + rn(D, scale=0.1), fn_b=rn(D, scale=0.1),
             mel_emb=rn(V, D, scale=0.05), mel_pos=rn(NMAX + 8, D, scale=0.05),
             codes=torch.randint(0, V - 2, (B, NMAX), generator=g, device=dev, dtype=torch.int32),
             state=torch.zeros(64, dtype=torch.int32, device=dev),
             x=rn(B, D), a=rn(B, D).to(torch.bfloat16), qkv=rn(B, 3 * D).to(torch.bfloat16),
             o=torch.zeros(B, D, dtype=torch.bfloat16, device=dev), h=rn(B, 4 * D).to(torch.bfloat16),
             hn=rn(B, D).to(torch.bfloat16), logits=torch.zeros(B, V, device=dev), prefix_kv=pfx[0], cand_kv=cand)
    t["state"][0] = STEP
    hd = lib.ArStep(B=B, D=D, H=H, L=L, V=V, P=PCAP, Nmax=NMAX, pos_mode=1, ld_codes=NMAX, attn_compact=compact,
                    groups=groups, row_start=rs, **t)
    first = [sum(sizes[:i]) for i in range(G)]
    return hd, t, dict(flat=flat, cand=cand, row=row, pfx=pfx, rs=rs, gidx=torch.tensor(gidx, device=dev), first=first, gen=g)


def _store_prompts(hd, t, w, Ps):
    """Poisons every group's whole prefix, stores a new random prompt of Ps[g] positions into it with
    ttb_ar_step_store_prefix_cap, and sets the group's P with ttb_ar_step_set_group_len. Checks the stored layout."""
    from tortoise_tts_b200 import lib
    pfx, g = w["pfx"], w["gen"]
    q = t["qkv"][:, :D].reshape(-1, H, 64)
    pfx[..., 0, :] = (4 * q[w["first"]]).unsqueeze(1).unsqueeze(3)          # keys that would dominate the group's first row
    pfx[..., 1, :] = POISON_V
    want = pfx.clone()
    for i, P in enumerate(Ps):
        for layer in range(L):
            qkv = torch.randn(P, 3 * D, generator=g, device="cuda").to(torch.bfloat16)
            lib.ar_step_store_prefix(qkv, P, H, pfx[i, layer], cap=PCAP)
            want[i, layer, :, :P, 0] = qkv[:, D:2 * D].reshape(P, H, 64).transpose(0, 1)
            want[i, layer, :, :P, 1] = qkv[:, 2 * D:].reshape(P, H, 64).transpose(0, 1)
        hd.set_group_len(i, P)
    torch.cuda.synchronize()
    assert torch.equal(pfx, want), "ttb_ar_step_store_prefix_cap wrote outside positions [0, P) or in another layout"


def _attn_ref(q, kn, vn, pk, pv, P_row, ck, cv, nold, more_prefix=0, more_cand=0):
    """float64 attention of one query per (row, head) over [prefix positions < P_row | own slots < nold | new token];
    more_*: attend that many positions past either bound (the mutants)."""
    ip = torch.arange(pk.shape[2], device=q.device)
    ic = torch.arange(ck.shape[2], device=q.device)
    sp = torch.einsum("nhd,nhtd->nht", q, pk).masked_fill(~(ip < (P_row + more_prefix)[:, None])[:, None], -torch.inf)
    sc = torch.einsum("nhd,nhtd->nht", q, ck).masked_fill(~(ic < (nold + more_cand)[:, None])[:, None], -torch.inf)
    s = torch.cat([sp, sc, (q * kn).sum(-1, keepdim=True)], dim=-1)
    return torch.einsum("nht,nhtd->nhd", torch.softmax(s, -1), torch.cat([pv, cv, vn.unsqueeze(2)], dim=2))


def _row_rel(got, want):
    n = got.shape[0]
    g, w = got.reshape(n, -1).double(), want.reshape(n, -1)
    return (g - w).abs().amax(1) / w.abs().amax(1).clamp_min(1e-6)


def _attention_launch(hd, t, w, P_row, shift, layers, label):
    """One attention launch at row_start = the J_CLASSES permutation `shift`, checked row by row."""
    cand, flat, B = w["cand"], w["flat"], t["qkv"].shape[0]
    rs = _row_starts(B, shift, STEP, J_CLASSES).cuda()
    w["rs"].copy_(rs)
    j = (STEP - rs).clamp(1, NMAX).long()
    slot = j - 1
    qkv = t["qkv"]
    q = qkv[:, :D].reshape(B, H, 64)
    stale = (torch.arange(NMAX, device="cuda")[None, :] >= slot[:, None])[:, None, :, None]     # [B, 1, NMAX, 1]
    flat.normal_(generator=w["gen"])             # fresh entries: the poison of an earlier launch may lie below j_b - 1
    for layer in range(L):
        cand[layer, ..., 0, :] = torch.where(stale, (4 * q).unsqueeze(2), cand[layer, ..., 0, :])
        cand[layer, ..., 1, :] = torch.where(stale, torch.full_like(cand[layer, ..., 1, :], POISON_V),
                                             cand[layer, ..., 1, :])
    before = flat.clone()
    t["o"].zero_()
    hd.step(phase_mask=PH_ATTN, layer_begin=layers[0], layer_end=layers[1])
    torch.cuda.synchronize()
    assert int(t["state"][2]) == 0, "internal time-out in the attention launch (%s)" % label
    assert int(t["state"][0]) == STEP, "the attention launch moved the shared step"
    # the append, and nothing else: slot j_b - 1 of every row, in every layer the launch ran
    want = before.clone()
    wc = want[w["row"]: w["row"] + cand.numel()].view_as(cand)
    rows = torch.arange(B, device="cuda")
    for layer in range(*layers):
        wc[layer, rows, :, slot, 0] = qkv[:, D:2 * D].reshape(B, H, 64)
        wc[layer, rows, :, slot, 1] = qkv[:, 2 * D:].reshape(B, H, 64)
        assert torch.equal(cand[layer, rows, :, slot], wc[layer, rows, :, slot]), "new K/V not in slot j_b - 1 (%s)" % label
    assert torch.equal(flat, want), "the attention wrote outside slot j_b - 1 of its rows (%s)" % label
    # the output of the last layer against float64, per row, and the two mutants
    layer = layers[1] - 1
    bc = before[w["row"]: w["row"] + cand.numel()].view_as(cand)[layer]
    worst, mut_p, mut_c = 0.0, [], []
    for r0 in range(0, B, 32):
        r = slice(r0, min(B, r0 + 32))
        gi = w["gidx"][r]
        pk, pv = (w["pfx"][gi, layer, :, :, i].double() for i in (0, 1))
        ck, cv = bc[r, :, :, 0].double(), bc[r, :, :, 1].double()
        qq = q[r].double() * 0.125
        kn, vn = qkv[r, D:2 * D].reshape(-1, H, 64).double(), qkv[r, 2 * D:].reshape(-1, H, 64).double()
        args = (qq, kn, vn, pk, pv, P_row[r], ck, cv, slot[r])
        ref = _attn_ref(*args)
        worst = max(worst, _row_rel(t["o"][r].reshape(-1, H, 64), ref).max().item())
        # control: a kernel that attended the first stale prefix position P_g (where the capacity leaves one) or the
        # first stale own slot would miss the bound by orders of magnitude on EVERY row
        m = P_row[r] < PCAP
        if m.any():
            mut_p.append(_row_rel(_attn_ref(*args, more_prefix=1)[m], ref[m]).min().item())
        mut_c.append(_row_rel(_attn_ref(*args, more_cand=1), ref).min().item())
    report("row_start attention %s" % label, worst)
    report("row_start attention %s, mutant attending prefix position P_g (least row error)" % label, min(mut_p))
    report("row_start attention %s, mutant attending slot j_b - 1 of the old cache (least row error)" % label, min(mut_c))
    assert min(mut_p) > 100 * ATTN_BOUND and min(mut_c) > 100 * ATTN_BOUND, "the poison would not show a stale read"
    assert worst < ATTN_BOUND, (label, worst)


@pytest.mark.parametrize("team", ["default", "one_warp"])
@pytest.mark.parametrize("kernel", list(KERNELS))
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_attention_rows_at_their_own_steps(layout, kernel, team):
    """The attention phase with row_start (ar_attn_only_kernel<true>, ar_attn_compact_kernel<true>, and the cooperative
    ar_step_kernel<true> over two layers): every row attends to [its group's first P_g prefix positions | its own slots
    0 .. j_b - 2 | the new token] with its own clamped j_b, writes the new K/V into slot j_b - 1 and nothing else. Prompts
    of 1 .. 352 positions are stored with ttb_ar_step_store_prefix_cap after setup; a second launch follows new prompts
    (some shorter, some longer) set with ttb_ar_step_set_group_len, and a new permutation of the row lengths."""
    compact, l0, l1 = KERNELS[kernel]
    sizes = LAYOUTS[layout]
    restore = _team(1 if team == "one_warp" else None)
    try:
        hd, t, w = _pool_step(sizes, compact, seed=len(sizes) + sum(sizes))
        G = len(sizes)
        for launch, (pshift, jshift) in enumerate(((0, 0), (2, 5))):
            Ps = [PROMPTS[(i + pshift) % len(PROMPTS)] for i in range(G)]
            if G == 2:                                  # the shared layouts: one short, one long prompt, then swapped
                Ps = [17, 352] if launch == 0 else [351, 13]
            _store_prompts(hd, t, w, Ps)
            P_row = torch.tensor(Ps, device="cuda")[w["gidx"]]
            _attention_launch(hd, t, w, P_row, jshift, (l0, l1), "%s %s team=%s launch %d" % (layout, kernel, team, launch))
    finally:
        restore()


@pytest.mark.parametrize("pos_mode", [0, 1])
@pytest.mark.parametrize("ld_codes", [37, NMAX])
def test_embed_rows(pos_mode, ld_codes):
    """ttb_ar_embed_step_rows at B = 256: x[b] = mel_emb[codes[b, j - 1]] + mel_pos[j + pos_mode] exactly, j = the row's
    own step clamped to [1, ld_codes]. codes and mel_pos sit inside guard regions of valid values."""
    from tortoise_tts_b200 import lib
    B, Dm, Vt, S, pad = 256, 1024, 300, 40, 1024
    g = torch.Generator(device="cuda")
    g.manual_seed(ld_codes + pos_mode)
    codes_all = torch.randint(0, Vt, (B * ld_codes + 2 * pad,), generator=g, device="cuda", dtype=torch.int32)
    codes = codes_all[pad: pad + B * ld_codes].view(B, ld_codes)
    mel_emb = torch.randn(Vt, Dm, generator=g, device="cuda")
    pos_all = torch.randn(1100 + 16, Dm, generator=g, device="cuda")
    mel_pos = pos_all[8:]
    classes = [1, ld_codes, 2, ABOVE, 16, ld_codes - 1, 17, BELOW, ld_codes + 1, 32, 0, 33]
    rs = _row_starts(B, 0, S, classes).cuda()
    state = torch.zeros(64, dtype=torch.int32, device="cuda")
    state[0] = S
    x = torch.full((B, Dm), float("nan"), device="cuda")
    lib.ar_embed_step(codes, ld_codes, state, mel_emb, mel_pos, B, Dm, pos_mode, x, row_start=rs)
    torch.cuda.synchronize()
    j = (S - rs).clamp(1, ld_codes).long()
    tok = codes[torch.arange(B, device="cuda"), j - 1].long()
    want = mel_emb[tok] + mel_pos[j + pos_mode]
    assert torch.equal(x, want), "rows %s" % (x != want).any(1).nonzero().flatten().tolist()[:8]
    assert int(state[0]) == S


SAMPLING = {"tts_defaults": (0.8, 50, 0.8, 2.0), "sharp": (0.3, 50, 0.95, 4.0)}


@pytest.mark.parametrize("params", list(SAMPLING))
def test_sampler_rows(params):
    """ttb_ar_sample_rows with ld_u < ld_codes: row b samples column c_b = clamp(step - row_start[b], 0,
    min(ld_codes, ld_u) - 1). Even rows hold two tokens of about equal mass and uniforms alternating 0.1 / 0.9 by column, so
    the column decides the token; odd rows hold random logits. Tokens against the float64 HF step, codes changed only at
    (b, c_b), seen / finished bookkeeping, finished rows write the stop token at c_b, the shared step advances once."""
    from tortoise_tts_b200 import lib
    temperature, top_k, top_p, rep = SAMPLING[params]
    B, LDC, LDU, S, pad = 256, 40, 29, 50, 64
    rng = np.random.default_rng(sorted(SAMPLING).index(params) + 31)
    classes = [0, 28, 1, ABOVE, 2, 29, 14, BELOW, 27, 35, 15, 39]       # 29 .. 39: past ld_u, inside ld_codes
    rs = _row_starts(B, 0, S, classes)
    col = (S - rs).clamp(0, min(LDC, LDU) - 1).long()
    ucols = np.arange(LDU)
    u = np.where((ucols[None, :] + np.arange(B)[:, None]) % 2 == 0, 0.1, 0.9).astype(np.float32)
    u[1::2] = rng.random((B // 2, LDU), dtype=np.float32)
    logits = (rng.standard_normal((B, V_SAMPLER), dtype=np.float32) * np.linspace(0.5, 4.0, B, dtype=np.float32)[:, None])
    pair = {}
    for b in range(0, B, 2):
        logits[b] = rng.standard_normal(V_SAMPLER).astype(np.float32) * 0.5 - 20.0
        a = STOP if b % 4 == 2 else int(rng.integers(2, 8000))
        c = int(rng.integers(2, 8000))
        while c == a:
            c = int(rng.integers(2, 8000))
        logits[b, a], logits[b, c] = 5.0, 4.875       # masses about 0.55 / 0.45 (0.6 / 0.4 at temperature 0.3)
        pair[b] = (a, c)
    seen_ids = []
    for b in range(B):
        s = {1, START} | set(int(i) for i in rng.integers(2, 8000, 5))
        s -= set(pair.get(b, ()))
        seen_ids.append(s)
    fin0 = torch.zeros(B, dtype=torch.int32)
    fin0[5::17] = 1
    seen = _seen_mask(seen_ids).cuda()
    seen_before = seen.clone()
    codes_all = torch.full((B * LDC + 2 * pad,), -1, dtype=torch.int32, device="cuda")
    codes = codes_all[pad: pad + B * LDC].view(B, LDC)
    u_all = torch.full((B * LDU + 2 * pad,), 0.5, device="cuda")
    u_all[pad: pad + B * LDU] = torch.from_numpy(u).cuda().reshape(-1)
    u_dev = u_all[pad: pad + B * LDU].view(B, LDU)
    finished = fin0.clone().cuda()
    state = torch.zeros(64, dtype=torch.int32, device="cuda")
    state[0] = S
    lib.ar_sample(torch.from_numpy(logits).cuda(), V_SAMPLER, V_SAMPLER, B, u_dev, LDU, seen, codes, LDC, finished, state,
                  temperature, top_k, top_p, rep, STOP, advance=True, row_start=rs.cuda())
    torch.cuda.synchronize()
    st = state.cpu()
    assert int(st[0]) == S + 1 and int(st[3]) == 0 and int(st[1]) == 0, st[:4]
    c = codes.cpu()
    drawn = c[torch.arange(B), col]
    want_codes = torch.full((B * LDC + 2 * pad,), -1, dtype=torch.int32)
    want_codes[pad: pad + B * LDC].view(B, LDC)[torch.arange(B), col] = drawn
    assert torch.equal(codes_all.cpu(), want_codes), "codes written outside column c_b"
    fin = finished.cpu()
    sb, sa = seen_before.cpu().numpy().view(np.uint32), seen.cpu().numpy().view(np.uint32)
    boundary = wrong_col = checked = 0
    for b in range(B):
        tok = int(drawn[b])
        if fin0[b]:
            assert tok == STOP and fin[b] == 1, b     # a finished row only writes the stop token
            continue
        want, wide, bnd = _hf_sample(logits[b], seen_ids[b], float(u[b, col[b]]), temperature, top_k, top_p, rep)
        if bnd:
            boundary += 1
            assert tok in wide, (b, tok, want)
        else:
            assert tok == want, (b, int(col[b]), tok, want)
        checked += 1
        exp = sb[b].copy()
        exp[tok >> 5] |= np.uint32(1 << (tok & 31))
        assert (sa[b] == exp).all(), "seen of row %d" % b
        assert int(fin[b]) == int(tok == STOP), "finished of row %d" % b
        if b in pair:
            assert tok in pair[b]
            # control: the neighbouring uniform column draws the other token of the pair
            for cn in (int(col[b]) - 1, int(col[b]) + 1):
                if 0 <= cn < LDU:
                    other = _hf_sample(logits[b], seen_ids[b], float(u[b, cn]), temperature, top_k, top_p, rep)[0]
                    assert other != tok and other in pair[b], (b, cn)
                    wrong_col += 1
    assert int(st[1]) == 0 and fin.sum() > fin0.sum(), "no row drew its stop token"
    report("row_start sampler %s: rows checked (boundary rows %d, neighbour-column controls %d)" %
           (params, boundary, wrong_col), checked)


def test_capture_rows():
    """ttb_ar_capture_latents_rows: row b writes column state.step - 1 - row_start[b] when it lies in [0, Nmax), equal
    to ttb_layernorm bit for bit and to float64 final_norm(ln_f(x)) within fp32 rounding; nothing else changes in an
    output of NaN canaries with ld_row > Nmax * D and guards in front of and behind the rows."""
    from tortoise_tts_b200 import lib
    B, Dm, NM, S = 256, 1024, 37, 60
    ld_row = NM * Dm + 260
    front, back = 64 * Dm, 1001 * Dm + ld_row
    g = torch.Generator(device="cuda")
    g.manual_seed(9)
    x = torch.randn(B, Dm, generator=g, device="cuda") * 2 + 0.5
    g1, b1 = 1 + 0.1 * torch.randn(Dm, generator=g, device="cuda"), 0.1 * torch.randn(Dm, generator=g, device="cuda")
    g2, b2 = 1 + 0.1 * torch.randn(Dm, generator=g, device="cuda"), 0.1 * torch.randn(Dm, generator=g, device="cuda")
    out_all = torch.full((front + B * ld_row + back,), float("nan"), device="cuda")
    out = out_all[front: front + B * ld_row]
    cols = [0, NM - 1, 1, ABOVE, 2, NM, 17, BELOW, NM - 2, -1, 33, 999]           # the row's step is column + 1
    rs = _row_starts(B, 0, S, [c if c in (ABOVE, BELOW) else c + 1 for c in cols]).cuda()
    state = torch.zeros(64, dtype=torch.int32, device="cuda")
    state[0] = S
    lib.ar_capture_latents(x, B, Dm, g1, b1, g2, b2, state, NM, out, ld_row, row_start=rs)
    ln = torch.empty(B, Dm, device="cuda")
    lib.layernorm(x, B, Dm, g1, b1, g2, b2, out_f32=ln)
    torch.cuda.synchronize()
    ref = F.layer_norm(F.layer_norm(x.double(), (Dm,), g1.double(), b1.double(), 1e-5), (Dm,), g2.double(), b2.double(), 1e-5)
    col = (S - 1 - rs).long().cpu()
    written = torch.zeros_like(out_all, dtype=torch.bool)
    worst, nw = 0.0, 0
    for b in range(B):
        c = int(col[b])
        if not 0 <= c < NM:
            continue
        o = front + b * ld_row + c * Dm
        got = out_all[o: o + Dm]
        written[o: o + Dm] = True
        assert torch.equal(got, ln[b]), "row %d column %d differs from ttb_layernorm" % (b, c)
        worst = max(worst, ((got.double() - ref[b]).abs().max() / ref[b].abs().max()).item())
        # control: a write one column off (either way) would leave column c at its NaN canary, and lands on canaries
        for n in (o - Dm, o + Dm):
            assert torch.isnan(out_all[n: n + Dm]).all()
        nw += 1
    assert nw > 0 and not torch.isnan(out_all[written]).any()
    assert torch.isnan(out_all[~written]).all(), "the capture wrote outside column step - 1 - row_start of its rows"
    report("row_start capture vs float64 final_norm(ln_f(x)) (%d rows written)" % nw, worst)
    assert worst < 1e-5


# ---------------------------------------------------------------- the slot workspace against the oracle
def _texts(lens, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(1, 255, (n - 5,), generator=g).tolist() + [0] for n in lens]     # prompt length n


def _run_pool(eng, C, N, plan, texts, voices, us, pos_mode):
    """Runs `plan` (("admit", slot, text) / ("advance", n) / ("release", slot)) on a slot workspace; returns one record
    (text, codes, captured latents) per admitted text, taken when it is released or at the end."""
    ws = eng.slot_workspace(C, N, pos_mode=pos_mode)
    occ, out = {}, []

    def take(s):
        n = min(ws.tokens(s), N - 1)            # a row past its cap keeps stepping; its last column is its own scratch
        out.append((occ.pop(s), ws.codes()[s, :n].clone(), ws.latents[s, :n].clone(), ws.tokens(s)))
    for ev in plan:
        if ev[0] == "admit":
            ws.admit(ev[1], voices[ev[2]], texts[ev[2]], us[ev[2]])
            occ[ev[1]] = ev[2]
        elif ev[0] == "advance":
            ws.advance(ev[1])
        else:
            take(ev[1])
            ws.release(ev[1])
    ws.check()
    for s in list(occ):
        take(s)
    return ws, out


def _vs_oracle(cfg, sd, out, texts, voices, pos_mode, label):
    from oracle import ar as oar
    sdc = {k: v.cuda().float() for k, v in sd.items()}
    worst = 0.0
    with torch.no_grad(), torch.device("cuda"):
        for u, codes, lat, _ in out:
            want = oar.stream_latents(sdc, cfg, voices[u].reshape(1, -1), texts[u], codes.long(), pos_mode)
            r = (lat - want).abs().max().item() / want.abs().max().item()
            report("slot workspace latents vs oracle %s text %d (%d tokens)" % (label, u, codes.numel()), r)
            worst = max(worst, r)
    assert worst < 0.03, (label, worst)                  # DESIGN §2: 3 % (bf16 tensor-core operands)


POOL_PLAN = [  # a long prompt and a short one at step 0, more texts at later steps, slot 0 reused by a shorter prompt
    ("admit", 0, 0), ("admit", -1, 1), ("advance", 9), ("admit", 1, 2), ("advance", 6), ("release", 0),
    ("admit", 0, 3), ("advance", 11), ("admit", 2, 4), ("advance", 4)]


@pytest.fixture(scope="module")
def medium():
    from tortoise_tts_b200.ar_engine import AREngine
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_autoregressive
    cfg = ModelConfig.medium()
    sd = synth_autoregressive(cfg, 0, False)
    return cfg, sd, AREngine(sd, cfg)


@pytest.mark.parametrize("pos_mode", ["ref_kv_quirk", "train_consistent"])
@pytest.mark.parametrize("mode,C", [("fused", 4), ("mixed", 24)])
def test_slot_workspace_vs_oracle(medium, pos_mode, mode, C):
    """Full width, two layers: texts admitted at global steps 0, 9 and 26, slot 0 reused by a 13-position prompt after
    a 352-position one, one row stepping past its cap of N = 30 tokens. Each row's captured latents against
    oracle.ar.stream_latents teacher-forced on that row's prompt and sampled codes."""
    from tortoise_tts_b200 import ar_engine
    cfg, sd, eng = medium
    E = ar_engine.AREngine
    texts = _texts([352, 17, 174, 13, 33], seed=4)
    g = torch.Generator().manual_seed(5)
    voices = [torch.randn(cfg.ar_dim, generator=g).cuda() for _ in texts]
    N = 30
    us = [torch.rand(N, generator=g).cuda() for _ in texts]
    plan = [(e[0], e[1] % C) + e[2:] if e[0] != "advance" else e for e in POOL_PLAN]
    saved = E.MODE
    E.MODE = mode
    try:
        ws, out = _run_pool(eng, C, N, plan, texts, voices, us, pos_mode)
        assert ws.st["mode"] == mode
    finally:
        E.MODE = saved
    assert any(n > N for *_, n in out), "no row stepped past its cap"
    _vs_oracle(cfg, sd, out, texts, voices, pos_mode, "%s C=%d %s" % (mode, C, pos_mode))


def test_slot_workspace_full_depth_vs_oracle():
    """30 layers, full width, three slots: texts admitted at steps 0 and 3, slot 0 reused by a shorter prompt at step 5;
    captured latents against the oracle."""
    from tortoise_tts_b200.ar_engine import AREngine
    from tortoise_tts_b200.config import ModelConfig
    from tortoise_tts_b200.synth import synth_autoregressive
    cfg = ModelConfig.full()
    sd = synth_autoregressive(cfg, 2, True)
    eng = AREngine(sd, cfg)
    texts = _texts([25, 62, 9], seed=6)
    g = torch.Generator().manual_seed(7)
    voices = [torch.randn(cfg.ar_dim, generator=g).cuda() for _ in texts]
    N = 12
    us = [torch.rand(N, generator=g).cuda() for _ in texts]
    plan = [("admit", 0, 0), ("advance", 3), ("admit", 1, 1), ("advance", 2), ("release", 0), ("admit", 0, 2),
            ("advance", 3)]
    _, out = _run_pool(eng, 3, N, plan, texts, voices, us, "ref_kv_quirk")
    _vs_oracle(cfg, sd, out, texts, voices, "ref_kv_quirk", "full depth")
