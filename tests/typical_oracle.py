"""TEST INFRASTRUCTURE ONLY (CPU oracle) — the sampling step of oracle/ar.py with the reference's typical-set filter.

`typical_sampling=True` puts `TypicalLogitsWarper(mass=typical_mass)` (tortoise/utils/typical_sampling.py:5-33) into the
custom logits-processor list of `UnifiedVoice.inference_speech` (autoregressive.py:558), which HF applies after its own
RepetitionPenaltyLogitsProcessor and before the Temperature / TopK / TopP warpers (stream_generator.py:946-947). The
warper in closed form, for one row of penalised scores s:

    logp = log_softmax(s), p = exp(logp), H = -nansum(p * logp), key_i = |-logp_i - H|
    T = {i : key_i <= v},  v = the smallest key with  sum_{key_j <= v} p_j >= mass

(`last_ind = (cumsum < mass).sum()`, `remove = sorted_key > sorted_key[last_ind]`: every key tied with v is kept, the
result does not depend on the sort order, T is never empty). Tokens outside T become -inf, so the top-k that follows
keeps min(top_k, |T|) tokens. Where the cumulative mass never reaches `mass` the reference indexes past the end and
raises; here everything is kept. With `typical_mass=None` both functions are oracle.ar's, unchanged.
"""
import torch

from oracle import ar


def typical_keep(s, mass):
    """Kept set T of TypicalLogitsWarper(mass) for scores s [V] (bool [V]) and the threshold key v."""
    logp = torch.log_softmax(s, dim=-1)
    p = torch.exp(logp)
    ent = -(logp * p).nansum()
    key = torch.abs(-logp - ent)
    sk, order = torch.sort(key, stable=True)
    cum = s[order].softmax(dim=-1).cumsum(dim=-1)
    last = min(int((cum < mass).sum()), s.numel() - 1)
    v = sk[last]
    return key <= v, float(v)


def sample_step(logits, prev_ids, u, temperature=0.8, top_k=50, top_p=0.8, repetition_penalty=2.0, typical_mass=None):
    """oracle.ar.sample_step with the typical filter between the repetition penalty and the temperature.
    Returns (token, kept_ids (desc), kept_probs)."""
    if typical_mass is None:
        return ar.sample_step(logits, prev_ids, u, temperature, top_k, top_p, repetition_penalty)
    s = logits.clone().float()
    idx = torch.tensor(sorted(set(int(i) for i in prev_ids)), dtype=torch.long)
    v = s[idx]
    s[idx] = torch.where(v < 0, v * repetition_penalty, v / repetition_penalty)
    keep, _ = typical_keep(s, typical_mass)
    s = s.masked_fill(~keep, float("-inf")) / temperature
    k = min(top_k, int(keep.sum()))
    vals, ids = torch.topk(s, k)
    p = torch.softmax(vals, dim=-1)
    excl = torch.cumsum(p, 0) - p
    kp_mask = excl < top_p
    kp_mask[0] = True
    kp = p[kp_mask]
    kp = kp / kp.sum()
    cdf = torch.cumsum(kp, 0)
    j = int(torch.searchsorted(cdf, torch.tensor(float(u)), right=True).clamp(max=kp.numel() - 1))
    return int(ids[kp_mask][j]), ids[kp_mask], kp


def generate(sd, cfg, cond_latent, text_tokens, uniforms, max_new, pos_mode="ref_kv_quirk", temperature=0.8, top_k=50,
             top_p=0.8, repetition_penalty=2.0, typical_mass=None):
    """oracle.ar.generate with `typical_mass`; returns codes [B, max_new] and the logits every step sampled from
    ([max_new, B, V], for kept-set checks)."""
    B = uniforms.shape[0]
    prompt = ar.prompt_embeddings(sd, cfg, cond_latent, text_tokens)
    start = sd["mel_embedding.weight"][cfg.start_mel_token] + sd["mel_pos_embedding.emb.weight"][0]
    emb = torch.cat([prompt, start.reshape(1, 1, -1)], dim=1).expand(B, -1, -1)
    hidden, past = ar.gpt2_trunk(sd, cfg, emb)
    logits = ar.mel_logits(sd, hidden[:, -1])
    codes = torch.full((B, max_new), cfg.stop_mel_token, dtype=torch.long)
    finished = [False] * B
    seen = [{1, cfg.start_mel_token} for _ in range(B)]
    trace = []
    for n in range(max_new):
        trace.append(logits.clone())
        toks = []
        for b in range(B):
            if finished[b]:
                toks.append(cfg.stop_mel_token)
                continue
            t, _, _ = sample_step(logits[b], seen[b], float(uniforms[b, n]), temperature, top_k, top_p,
                                  repetition_penalty, typical_mass)
            toks.append(t)
            seen[b].add(t)
            if t == cfg.stop_mel_token:
                finished[b] = True
        codes[:, n] = torch.tensor(toks)
        if all(finished) or n == max_new - 1:
            break
        ids = torch.tensor(toks, dtype=torch.long)
        e = sd["mel_embedding.weight"][ids] + sd["mel_pos_embedding.emb.weight"][ar.mel_pos_index(n + 1, pos_mode)]
        hidden, past = ar.gpt2_trunk(sd, cfg, e.unsqueeze(1), past)
        logits = ar.mel_logits(sd, hidden[:, -1])
    return codes, torch.stack(trace)
