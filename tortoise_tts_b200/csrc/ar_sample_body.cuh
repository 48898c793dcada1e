// The body of the fused sampler kernels of csrc/ar.cu (ar_sample_kernel<TYPICAL> and ar_sample_params_kernel), included
// as text inside each kernel. In scope there: the kernel's pointer and size parameters, `SRC` (a constexpr SampSrc) and
// the settings temperature, top_k, top_p, rep_penalty, typical_mass. A __forceinline__ function in its place gives
// ar_sample_kernel<true> different instructions: the optimiser sees one more inlining level and hoists differently.
  extern __shared__ float sval[];           // V floats: processed scores
  __shared__ int hist[256];
  __shared__ uint32_t s_prefix;
  __shared__ int s_remaining;
  __shared__ int s_eq;                      // elements whose key equals the threshold key (known after the last pass)
  __shared__ float cand_v[SAMP_CAP];
  __shared__ int cand_i[SAMP_CAP];
  __shared__ int s_ncand;
  const int b = blockIdx.x;
  const bool typical = SRC == SampSrc::SCALAR_TYPICAL || (SRC == SampSrc::TABLE && typical_mass > 0.f);
  const int gstep = state->step;
  // the column this row samples: the shared step, or with row_start the row's own step clamped to the rows of codes and
  // uniforms (include/ttb.h)
  const int step = row_start ? min(max(gstep - row_start[b], 0), min(ld_codes, ld_u) - 1) : gstep;
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
    sval[i] = typical ? s : s / temperature;  // the typical filter sees the scores before temperature, then divides
  }
  int kk = min(top_k, V);                   // top-k over the candidates: the whole row, or T with the typical filter
  if constexpr (SRC != SampSrc::SCALAR) {
    __shared__ unsigned long long t_hist[256];
    __shared__ unsigned long long t_rem;
    __shared__ float t_red[32];
    __shared__ int t_count;
    if (typical) {
      __syncthreads();
      // masked tokens are -inf, the lowest keys of all: with k <= |T| the select, the tie fill and every fallback of the
      // draw only ever see tokens of T
      kk = min(kk, typical_filter(sval, V, temperature, typical_mass, t_hist, t_red, &s_prefix, &t_rem, &t_count));
    }
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
        state->step = gstep + 1;
      }
    }
  }
