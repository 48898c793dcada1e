// Autoregressive sampler support kernels (UnifiedVoice / GPT2InferenceModel hot loop):
// embedding gathers, the fused HF sample() step and the post-processing of generated codes.
#include "common.cuh"
#include "ttb_internal.h"

namespace ttb {

__global__ void embed_kernel(const int* __restrict__ ids, const int* __restrict__ pos, int n, int D,
                             const float* __restrict__ table, const float* __restrict__ pos_table,
                             float* __restrict__ out) {
  const int r = blockIdx.x;
  const float* t = table + (long long)ids[r] * D;
  const float* p = (pos_table && pos) ? pos_table + (long long)pos[r] * D : nullptr;
  for (int c = threadIdx.x; c < D; c += blockDim.x) out[(long long)r * D + c] = t[c] + (p ? p[c] : 0.f);
}

__global__ void ar_embed_step_kernel(const int* __restrict__ codes, int ld_codes, const TtbArState* __restrict__ state,
                                     const float* __restrict__ mel_emb, const float* __restrict__ mel_pos, int D,
                                     int pos_mode, float* __restrict__ x) {
  const int b = blockIdx.x;
  const int j = state->step;                 // index of this token inside the mel segment (start token = 0)
  const int tok = codes[(long long)b * ld_codes + j - 1];
  const int pos = pos_mode ? j + 1 : j;      // autoregressive.py:147-149 (SURVEY App. D-1)
  const float* t = mel_emb + (long long)tok * D;
  const float* p = mel_pos + (long long)pos * D;
  for (int c = threadIdx.x; c < D; c += blockDim.x) x[(long long)b * D + c] = t[c] + p[c];
}

// ------------------------------------------------------------------ fused sampler
// One block (256 threads) per candidate. Radix-select of the top_k-th largest value (4 passes of 8 bits over the
// order-preserving uint32 image of the float), gather of the survivors (<= CAP), bitonic sort by one warp,
// softmax, top-p cut on the exclusive prefix mass, inverse-CDF draw. The TYPICAL instantiation first restricts the
// row to the typical set (typical_filter below), between the repetition penalty and the temperature.
constexpr int SAMP_THREADS = 256;
constexpr int SAMP_CAP = 64;

TTB_DEVINL uint32_t f2key(float f) {
  uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// ---- typical-set filter (TypicalLogitsWarper, reference tortoise/utils/typical_sampling.py:11-33), on the penalised
// scores s before temperature: logp = log_softmax(s), H = -nansum(p logp), key_i = |-logp_i - H|; kept set
// T = {i : key_i <= v}, v = the smallest key with sum_{key_j <= v} p_j >= mass (ties at v all kept, never empty).
// key_i and p_i are recomputed from sval wherever they are needed instead of being stored: a second V-float array
// would take the dynamic shared memory past 48 KB (opt-in attribute) and halve the blocks per SM, while recomputing is
// a few instructions per element and pass. The recomputation uses the same rounded operations everywhere (__fsub_rn /
// __fadd_rn cannot be contracted), so every pass sees bit-identical keys and masses.
constexpr double TYP_QSCALE = 1099511627776.0;   // 2^40: p in [0, 1] as 64-bit fixed point (bin sums cannot overflow)

TTB_DEVINL float typ_logp(float s, float m, float lz) { return __fsub_rn(__fsub_rn(s, m), lz); }  // (s - max) - logZ
TTB_DEVINL uint32_t typ_key(float lp, float H) { return f2key(fabsf(__fadd_rn(lp, H))); }       // |-logp - H|
TTB_DEVINL unsigned long long typ_q(float lp) { return __float2ull_rn(__fmul_rn(expf(lp), (float)TYP_QSCALE)); }

// Leaves sval[i] = s_i / temperature for i in T and -inf elsewhere; returns |T| (>= 1). hist: 256 u64 of shared memory,
// red: 32 floats. The bin masses are sums of integers, so the result does not depend on the order of the atomics.
TTB_DEVINL int typical_filter(float* sval, int V, float temperature, float mass, unsigned long long* hist, float* red,
                              uint32_t* s_prefix, unsigned long long* s_rem, int* s_count) {
  float m = -INFINITY;
  for (int i = threadIdx.x; i < V; i += SAMP_THREADS) m = fmaxf(m, sval[i]);
  m = block_max(m, red);
  float z = 0.f;
  for (int i = threadIdx.x; i < V; i += SAMP_THREADS) z += expf(sval[i] - m);
  const float lz = logf(block_sum(z, red));
  float h = 0.f;
  for (int i = threadIdx.x; i < V; i += SAMP_THREADS) {
    const float lp = typ_logp(sval[i], m, lz);
    const float t = expf(lp) * lp;
    if (!isnan(t)) h += t;                  // nansum
  }
  const float H = -block_sum(h, red);
  if (threadIdx.x == 0) { *s_prefix = 0; *s_count = 0; }
  // radix select over the keys in ASCENDING order, weighted by mass: 4 passes of 8 bits; in each, the bin where the
  // cumulative mass of the keys below it (within the current prefix) first reaches the remaining target
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    hist[threadIdx.x] = 0ull;
    __syncthreads();
    const uint32_t prefix = *s_prefix;
    const uint32_t mask = (pass == 0) ? 0u : (0xFFFFFFFFu << (shift + 8));
    for (int base = 0; base < V; base += SAMP_THREADS) {          // uniform trip count: every lane takes part
      const int i = base + threadIdx.x;
      int bin = 256;
      unsigned long long q = 0ull;
      if (i < V) {
        const float lp = typ_logp(sval[i], m, lz);
        const uint32_t k = typ_key(lp, H);
        if ((k & mask) == prefix) { bin = (int)((k >> shift) & 255u); q = typ_q(lp); }
      }
      if (bin < 256) atomicAdd(&hist[bin], q);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      // bins in ascending key order: the first whose cumulative mass reaches the remaining target
      unsigned long long r = *s_rem;
      if (pass == 0) {
        unsigned long long total = 0ull;
        for (int d = 0; d < 256; ++d) total += hist[d];
        // sum_{key <= v} p >= mass, measured against the total so that mass = 1 keeps everything
        r = (unsigned long long)ceil((double)mass * (double)total);
        r = max(1ull, min(r, total));
      }
      int d = 0;
      for (; d < 255; ++d) {
        const unsigned long long hd = hist[d];
        if (hd >= r) break;
        r -= hd;
      }
      *s_prefix = prefix | ((uint32_t)d << shift);
      *s_rem = r;
    }
    __syncthreads();
  }
  const uint32_t v = *s_prefix;
  int n = 0;
  for (int i = threadIdx.x; i < V; i += SAMP_THREADS) {
    const float s = sval[i];
    const bool in = typ_key(typ_logp(s, m, lz), H) <= v;
    sval[i] = in ? s / temperature : -INFINITY;
    n += in ? 1 : 0;
  }
  atomicAdd(s_count, n);
  __syncthreads();
  return *s_count;
}

template <bool TYPICAL>
__global__ void __launch_bounds__(SAMP_THREADS)
ar_sample_kernel(const float* __restrict__ logits, int ld_logits, int V, const float* __restrict__ uniforms, int ld_u,
                 uint32_t* __restrict__ seen, int* __restrict__ codes, int ld_codes, int* __restrict__ finished,
                 TtbArState* __restrict__ state, float temperature, int top_k, float top_p, float rep_penalty,
                 int stop_token, int advance, float typical_mass) {
  extern __shared__ float sval[];           // V floats: processed scores
  __shared__ int hist[256];
  __shared__ uint32_t s_prefix;
  __shared__ int s_remaining;
  __shared__ int s_eq;                      // elements whose key equals the threshold key (known after the last pass)
  __shared__ float cand_v[SAMP_CAP];
  __shared__ int cand_i[SAMP_CAP];
  __shared__ int s_ncand;
  const int b = blockIdx.x;
  const int step = state->step;
  const int words = (V + 31) >> 5;
  const int lane = threadIdx.x & 31;
  uint32_t* myseen = seen + (long long)b * words;
  const float* lrow = logits + (long long)b * ld_logits;
  if (finished[b]) {
    // HF: finished rows keep emitting pad_token_id (= stop token) (stream_generator.py:974-981)
    if (threadIdx.x == 0) codes[(long long)b * ld_codes + step] = stop_token;
  } else {
  for (int i = threadIdx.x; i < V; i += SAMP_THREADS) {
    float s = lrow[i];
    if ((myseen[i >> 5] >> (i & 31)) & 1u) s = (s < 0.f) ? s * rep_penalty : s / rep_penalty;
    sval[i] = TYPICAL ? s : s / temperature;  // the typical filter sees the scores before temperature, then divides
  }
  int kk = min(top_k, V);                   // top-k over the candidates: the whole row, or T with the typical filter
  if constexpr (TYPICAL) {
    __shared__ unsigned long long t_hist[256];
    __shared__ unsigned long long t_rem;
    __shared__ float t_red[32];
    __shared__ int t_count;
    __syncthreads();
    // masked tokens are -inf, the lowest keys of all: with k <= |T| the select, the tie fill and every fallback of the
    // draw only ever see tokens of T
    kk = min(kk, typical_filter(sval, V, temperature, typical_mass, t_hist, t_red, &s_prefix, &t_rem, &t_count));
  }
  if (threadIdx.x == 0) { s_prefix = 0; s_remaining = kk; s_ncand = 0; }
  __syncthreads();
  // radix select: find key T of the k-th largest element. The histogram updates are aggregated per warp (the keys of a
  // logit row share their exponent byte: unaggregated, pass 0 is ~8000 atomics on two or three shared-memory words), and
  // the bin scan is done by one warp (8 bins per lane + a suffix scan) instead of a 256-step loop of one thread.
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    hist[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t prefix = s_prefix;
    const uint32_t mask = (pass == 0) ? 0u : (0xFFFFFFFFu << (shift + 8));
    for (int base = 0; base < V; base += SAMP_THREADS) {          // uniform trip count: every lane takes part in the match
      const int i = base + threadIdx.x;
      int bin = 256;
      if (i < V) {
        const uint32_t k = f2key(sval[i]);
        if ((k & mask) == prefix) bin = (int)((k >> shift) & 255u);
      }
      const unsigned peers = __match_any_sync(0xffffffffu, bin);
      if (bin < 256 && lane == __ffs(peers) - 1) atomicAdd(&hist[bin], __popc(peers));
    }
    __syncthreads();
    if (threadIdx.x < 32) {
      // bins 255 .. 0 in descending order: the bin d with  sum(hist[d+1 ..]) < remaining <= sum(hist[d ..])
      int h[8];
      int mine = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) { h[j] = hist[lane * 8 + j]; mine += h[j]; }
      int above = mine;                     // inclusive suffix sum over the lanes (lane 31 = the highest bins)
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_down_sync(0xffffffffu, above, o); if (lane + o < 32) above += t; }
      above -= mine;                        // elements in bins above this lane's
      const int rem = s_remaining;
      const bool here = (above < rem) && (rem <= above + mine);
      const unsigned found = __ballot_sync(0xffffffffu, here);
      if (found) {
        if (here) {
          int r = rem - above, d = 7;
          for (; d > 0; --d) {
            if (h[d] >= r) break;
            r -= h[d];
          }
          s_prefix = prefix | ((uint32_t)(lane * 8 + d) << shift);
          s_remaining = r;
          s_eq = h[d];
        }
      } else if (lane == 0) {               // fewer matching elements than requested (cannot happen for top_k <= V)
        s_prefix = prefix;
        s_remaining = rem - (above + mine - h[0]);
        s_eq = h[0];
      }
    }
    __syncthreads();
  }
  const uint32_t thr = s_prefix;  // key of the k-th largest; HF keeps everything >= it (ties included)
  const int n_ge = (kk - s_remaining) + s_eq;              // elements with key >= thr
  if (n_ge <= SAMP_CAP) {
    // the common case: everything that is kept fits; slot order is irrelevant (sorted below by value, then index)
    for (int i = threadIdx.x; i < V; i += SAMP_THREADS) {
      const float s = sval[i];
      if (f2key(s) >= thr) {
        const int slot = atomicAdd(&s_ncand, 1);
        cand_v[slot] = s; cand_i[slot] = i;
      }
    }
    __syncthreads();
  } else {
  // values strictly above the threshold: at most top_k - 1 < SAMP_CAP of them, slot order is irrelevant (sorted below)
  for (int i = threadIdx.x; i < V; i += SAMP_THREADS) {
    const float s = sval[i];
    if (f2key(s) > thr) {
      const int slot = atomicAdd(&s_ncand, 1);
      cand_v[slot] = s; cand_i[slot] = i;
    }
  }
  __syncthreads();
  // values equal to the threshold, in ASCENDING INDEX order (one warp, ballot compaction): if more than SAMP_CAP values
  // tie (flat logits, duplicated mel_head rows) the survivors are the lowest ids - a fixed set, not a race
  if (threadIdx.x < 32) {
    int n = s_ncand;
    for (int base = 0; base < V && n < SAMP_CAP; base += 32) {
      const int i = base + threadIdx.x;
      const bool tie = (i < V) && (f2key(sval[i]) == thr);
      const unsigned m = __ballot_sync(0xffffffffu, tie);
      if (tie) {
        const int slot = n + __popc(m & ((1u << threadIdx.x) - 1u));
        if (slot < SAMP_CAP) { cand_v[slot] = sval[i]; cand_i[slot] = i; }
      }
      n += __popc(m);
    }
    if (threadIdx.x == 0) s_ncand = n;
  }
  __syncthreads();
  }
  if (threadIdx.x < 32) {
    const int n = min(s_ncand, SAMP_CAP);
    // two elements per lane; bitonic sort of 64, descending by value then ascending by index
    float v0 = (lane < n) ? cand_v[lane] : -INFINITY, v1 = (lane + 32 < n) ? cand_v[lane + 32] : -INFINITY;
    int i0 = (lane < n) ? cand_i[lane] : 0x7fffffff, i1 = (lane + 32 < n) ? cand_i[lane + 32] : 0x7fffffff;
    __syncwarp();
    cand_v[lane] = v0; cand_v[lane + 32] = v1; cand_i[lane] = i0; cand_i[lane + 32] = i1;
    __syncwarp();
    for (int k = 2; k <= 64; k <<= 1) {
      for (int j = k >> 1; j > 0; j >>= 1) {
        for (int e = lane; e < 64; e += 32) {
          const int partner = e ^ j;
          if (partner > e) {
            const bool desc = ((e & k) == 0);
            const float a = cand_v[e], c = cand_v[partner];
            const int ia = cand_i[e], ic = cand_i[partner];
            const bool a_before = (a > c) || (a == c && ia < ic);  // a should precede c in descending order
            if (desc ? !a_before : a_before) {
              cand_v[e] = c; cand_v[partner] = a; cand_i[e] = ic; cand_i[partner] = ia;
            }
          }
        }
        __syncwarp();
      }
    }
    // softmax over the survivors (descending), top-p on exclusive prefix mass
    const float vmax = cand_v[0];
    float p0 = (lane < n) ? __expf(cand_v[lane] - vmax) : 0.f;
    float p1 = (lane + 32 < n) ? __expf(cand_v[lane + 32] - vmax) : 0.f;
    const float tot = warp_sum(p0 + p1);
    p0 /= tot; p1 /= tot;
    // inclusive scan over 64 entries in order (lane, then lane+32)
    float c0 = p0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { float t = __shfl_up_sync(0xffffffffu, c0, o); if (lane >= o) c0 += t; }
    const float first_half = __shfl_sync(0xffffffffu, c0, 31);
    float c1 = p1;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { float t = __shfl_up_sync(0xffffffffu, c1, o); if (lane >= o) c1 += t; }
    c1 += first_half;
    const bool keep0 = (lane < n) && ((c0 - p0) < top_p || lane == 0);
    const bool keep1 = (lane + 32 < n) && ((c1 - p1) < top_p);
    const float kept = warp_sum((keep0 ? p0 : 0.f) + (keep1 ? p1 : 0.f));
    // draw: smallest index with cumulative kept mass / kept > u (kept set is a prefix of the sorted list)
    const float u = uniforms[(long long)b * ld_u + step] * kept;
    const unsigned m0 = __ballot_sync(0xffffffffu, keep0 && c0 > u);
    const unsigned m1 = __ballot_sync(0xffffffffu, keep1 && c1 > u);
    const unsigned k0m = __ballot_sync(0xffffffffu, keep0);
    const unsigned k1m = __ballot_sync(0xffffffffu, keep1);
    int pick;
    if (m0) pick = __ffs(m0) - 1;
    else if (m1) pick = 32 + __ffs(m1) - 1;
    else pick = k1m ? 32 + (31 - __clz(k1m)) : (31 - __clz(k0m));  // numerical slack: last kept
    if (lane == 0) {
      const int tok = cand_i[pick];
      codes[(long long)b * ld_codes + step] = tok;
      myseen[tok >> 5] |= (1u << (tok & 31));
      if (tok == stop_token) finished[b] = 1;
    }
  }
  }   // !finished[b]
  if (advance) {
    // the last block to get here advances the step counter (every block read it at its start) and refreshes the
    // all-finished flag: what the separate ar_sample_advance_kernel launch did, without the launch
    __shared__ int s_last;
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      s_last = (atomicAdd(&state->reserved[1], 1) == (int)gridDim.x - 1);
    }
    __syncthreads();
    if (s_last) {
      __threadfence();
      int unf = 0;
      for (int i = threadIdx.x; i < (int)gridDim.x; i += SAMP_THREADS) unf |= (__ldcg(finished + i) == 0);
      unf = __syncthreads_or(unf);
      if (threadIdx.x == 0) {
        state->reserved[1] = 0;
        state->all_finished = unf ? 0 : 1;
        state->step = step + 1;
      }
    }
  }
}

// fix_autoregressive_output (api.py:87-114) + calm trim (api.py:547-556); one thread per row (rows are short)
__global__ void ar_fix_codes_kernel(int* __restrict__ codes, int B, int L, int stop_token, int* __restrict__ trim_len) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  int* c = codes + (long long)b * L;
  int stm = -1;
  for (int i = 0; i < L; ++i) if (c[i] == stop_token) { stm = i; break; }
  if (stm >= 0) {
    for (int i = stm; i < L; ++i) c[i] = 83;
    if (L >= 3) { c[L - 3] = 45; c[L - 2] = 45; c[L - 1] = 248; }
  }
  int run = 0, cut = L;
  for (int i = 0; i < L; ++i) {
    run = (c[i] == 83) ? run + 1 : 0;
    if (run > 8) { cut = i; break; }
  }
  if (trim_len) trim_len[b] = cut;
}

}  // namespace ttb
using namespace ttb;

extern "C" int ttb_embed(const int* ids, const int* pos, int n, int D, const float* table, const float* pos_table,
                         float* out, void* stream) {
  if (n <= 0) return 0;
  embed_kernel<<<n, 256, 0, static_cast<cudaStream_t>(stream)>>>(ids, pos, n, D, table, pos_table, out);
  TTB_CHECK_LAUNCH("embed_kernel");
  return 0;
}

extern "C" int ttb_ar_embed_step(const int* codes, int ld_codes, const TtbArState* state, const float* mel_emb,
                                 const float* mel_pos, int B, int D, int pos_mode, float* x, void* stream) {
  ar_embed_step_kernel<<<B, 256, 0, static_cast<cudaStream_t>(stream)>>>(codes, ld_codes, state, mel_emb, mel_pos, D,
                                                                        pos_mode, x);
  TTB_CHECK_LAUNCH("ar_embed_step_kernel");
  return 0;
}

template <bool TYPICAL>
static int launch_ar_sample(const char* name, const float* logits, int ld_logits, int V, int B, const float* uniforms,
                            int ld_u, uint32_t* seen, int* codes, int ld_codes, int* finished, TtbArState* state,
                            float temperature, int top_k, float top_p, float rep_penalty, int stop_token, int advance,
                            float typical_mass, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (top_k <= 0 || top_k > 50) { set_error("%s: top_k=%d unsupported (1..50)", name, top_k); return -1; }
  const size_t smem = (size_t)V * sizeof(float);
  if (smem > 40 * 1024) { set_error("%s: vocabulary %d too large", name, V); return -1; }
  ar_sample_kernel<TYPICAL><<<B, SAMP_THREADS, smem, st>>>(logits, ld_logits, V, uniforms, ld_u, seen, codes, ld_codes,
                                                           finished, state, temperature, top_k, top_p, rep_penalty,
                                                           stop_token, advance ? 1 : 0, typical_mass);
  TTB_CHECK_LAUNCH("ar_sample_kernel");
  return 0;
}

extern "C" int ttb_ar_sample(const float* logits, int ld_logits, int V, int B, const float* uniforms, int ld_u,
                             uint32_t* seen, int* codes, int ld_codes, int* finished, TtbArState* state,
                             float temperature, int top_k, float top_p, float rep_penalty, int stop_token, int advance,
                             void* stream) {
  return launch_ar_sample<false>("ttb_ar_sample", logits, ld_logits, V, B, uniforms, ld_u, seen, codes, ld_codes,
                                 finished, state, temperature, top_k, top_p, rep_penalty, stop_token, advance, 1.f,
                                 stream);
}

extern "C" int ttb_ar_sample_typical(const float* logits, int ld_logits, int V, int B, const float* uniforms, int ld_u,
                                     uint32_t* seen, int* codes, int ld_codes, int* finished, TtbArState* state,
                                     float temperature, int top_k, float top_p, float rep_penalty, int stop_token,
                                     int advance, float typical_mass, void* stream) {
  if (!(typical_mass > 0.f && typical_mass <= 1.f)) {
    set_error("ttb_ar_sample_typical: typical_mass=%g outside (0, 1]", (double)typical_mass);
    return -1;
  }
  return launch_ar_sample<true>("ttb_ar_sample_typical", logits, ld_logits, V, B, uniforms, ld_u, seen, codes, ld_codes,
                                finished, state, temperature, top_k, top_p, rep_penalty, stop_token, advance,
                                typical_mass, stream);
}

extern "C" int ttb_ar_fix_codes(int* codes, int B, int L, int stop_token, int* trim_len, void* stream) {
  ar_fix_codes_kernel<<<(B + 63) / 64, 64, 0, static_cast<cudaStream_t>(stream)>>>(codes, B, L, stop_token, trim_len);
  TTB_CHECK_LAUNCH("ar_fix_codes_kernel");
  return 0;
}
