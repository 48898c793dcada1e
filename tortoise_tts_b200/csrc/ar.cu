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
                                     const int* __restrict__ row_start, const float* __restrict__ mel_emb,
                                     const float* __restrict__ mel_pos, int D, int pos_mode, float* __restrict__ x) {
  const int b = blockIdx.x;
  // index of this token inside the mel segment (start token = 0); with row_start, the row's own step clamped to
  // [1, ld_codes] (include/ttb.h)
  int j = state->step;
  if (row_start) j = min(max(j - row_start[b], 1), ld_codes);
  const int tok = codes[(long long)b * ld_codes + j - 1];
  const int pos = pos_mode ? j + 1 : j;      // autoregressive.py:147-149 (SURVEY App. D-1)
  const float* t = mel_emb + (long long)tok * D;
  const float* p = mel_pos + (long long)pos * D;
  for (int c = threadIdx.x; c < D; c += blockDim.x) x[(long long)b * D + c] = t[c] + p[c];
}

// ------------------------------------------------------------------ fused sampler
// One block (256 threads) per candidate. Radix-select of the top_k-th largest value (4 passes of 8 bits over the
// order-preserving uint32 image of the float), gather of the survivors (<= CAP), bitonic sort by one warp,
// softmax, top-p cut on the exclusive prefix mass, inverse-CDF draw. With the typical filter on, the row is first
// restricted to the typical set (typical_filter below), between the repetition penalty and the temperature. One body
// (ar_sample_body.cuh) serves the scalar-settings kernels and the per-row-settings kernel.
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

// Where the sampler's settings come from: the launch's scalar parameters, with the typical filter off (SCALAR) or on
// (SCALAR_TYPICAL), or the row's entry of a TtbSampleParams table (TABLE: the filter is on where typical_mass > 0; the
// branch depends on blockIdx.x only, so it is uniform across the block).
enum class SampSrc { SCALAR, SCALAR_TYPICAL, TABLE };

template <bool TYPICAL>
__global__ void __launch_bounds__(SAMP_THREADS)
ar_sample_kernel(const float* __restrict__ logits, int ld_logits, int V, const float* __restrict__ uniforms, int ld_u,
                 uint32_t* __restrict__ seen, int* __restrict__ codes, int ld_codes, int* __restrict__ finished,
                 TtbArState* __restrict__ state, float temperature, int top_k, float top_p, float rep_penalty,
                 int stop_token, int advance, float typical_mass, const int* __restrict__ row_start) {
  constexpr SampSrc SRC = TYPICAL ? SampSrc::SCALAR_TYPICAL : SampSrc::SCALAR;
#include "ar_sample_body.cuh"
}

// The sampler with row b's settings read from params[b] (a device table, not the kernel-parameter space). top_k is
// clamped to [1, 50] here so that a bad table cannot write past the SAMP_CAP candidate slots; the host validates it.
__global__ void __launch_bounds__(SAMP_THREADS)
ar_sample_params_kernel(const float* __restrict__ logits, int ld_logits, int V, const float* __restrict__ uniforms,
                        int ld_u, uint32_t* __restrict__ seen, int* __restrict__ codes, int ld_codes,
                        int* __restrict__ finished, TtbArState* __restrict__ state,
                        const TtbSampleParams* __restrict__ params, int stop_token, int advance,
                        const int* __restrict__ row_start) {
  constexpr SampSrc SRC = SampSrc::TABLE;
  const TtbSampleParams prm = params[blockIdx.x];
  const float temperature = prm.temperature, top_p = prm.top_p, rep_penalty = prm.rep_penalty;
  const float typical_mass = prm.typical_mass;
  const int top_k = min(max(prm.top_k, 1), 50);
#include "ar_sample_body.cuh"
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

extern "C" int ttb_ar_embed_step_rows(const int* codes, int ld_codes, const TtbArState* state, const int* row_start,
                                      const float* mel_emb, const float* mel_pos, int B, int D, int pos_mode, float* x,
                                      void* stream) {
  ar_embed_step_kernel<<<B, 256, 0, static_cast<cudaStream_t>(stream)>>>(codes, ld_codes, state, row_start, mel_emb,
                                                                        mel_pos, D, pos_mode, x);
  TTB_CHECK_LAUNCH("ar_embed_step_kernel");
  return 0;
}

extern "C" int ttb_ar_embed_step(const int* codes, int ld_codes, const TtbArState* state, const float* mel_emb,
                                 const float* mel_pos, int B, int D, int pos_mode, float* x, void* stream) {
  return ttb_ar_embed_step_rows(codes, ld_codes, state, nullptr, mel_emb, mel_pos, B, D, pos_mode, x, stream);
}

template <bool TYPICAL>
static int launch_ar_sample(const char* name, const float* logits, int ld_logits, int V, int B, const float* uniforms,
                            int ld_u, uint32_t* seen, int* codes, int ld_codes, int* finished, TtbArState* state,
                            float temperature, int top_k, float top_p, float rep_penalty, int stop_token, int advance,
                            float typical_mass, const int* row_start, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (top_k <= 0 || top_k > 50) { set_error("%s: top_k=%d unsupported (1..50)", name, top_k); return -1; }
  const size_t smem = (size_t)V * sizeof(float);
  if (smem > 40 * 1024) { set_error("%s: vocabulary %d too large", name, V); return -1; }
  if (row_start && (ld_codes <= 0 || ld_u <= 0)) { set_error("%s: row_start needs ld_codes, ld_u > 0", name); return -1; }
  ar_sample_kernel<TYPICAL><<<B, SAMP_THREADS, smem, st>>>(logits, ld_logits, V, uniforms, ld_u, seen, codes, ld_codes,
                                                           finished, state, temperature, top_k, top_p, rep_penalty,
                                                           stop_token, advance ? 1 : 0, typical_mass, row_start);
  TTB_CHECK_LAUNCH("ar_sample_kernel");
  return 0;
}

extern "C" int ttb_ar_sample(const float* logits, int ld_logits, int V, int B, const float* uniforms, int ld_u,
                             uint32_t* seen, int* codes, int ld_codes, int* finished, TtbArState* state,
                             float temperature, int top_k, float top_p, float rep_penalty, int stop_token, int advance,
                             void* stream) {
  return launch_ar_sample<false>("ttb_ar_sample", logits, ld_logits, V, B, uniforms, ld_u, seen, codes, ld_codes,
                                 finished, state, temperature, top_k, top_p, rep_penalty, stop_token, advance, 1.f,
                                 nullptr, stream);
}

extern "C" int ttb_ar_sample_rows(const float* logits, int ld_logits, int V, int B, const float* uniforms, int ld_u,
                                  uint32_t* seen, int* codes, int ld_codes, int* finished, TtbArState* state,
                                  float temperature, int top_k, float top_p, float rep_penalty, int stop_token, int advance,
                                  const int* row_start, void* stream) {
  return launch_ar_sample<false>("ttb_ar_sample_rows", logits, ld_logits, V, B, uniforms, ld_u, seen, codes, ld_codes,
                                 finished, state, temperature, top_k, top_p, rep_penalty, stop_token, advance, 1.f,
                                 row_start, stream);
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
                                typical_mass, nullptr, stream);
}

extern "C" int ttb_ar_sample_params(const float* logits, int ld_logits, int V, int B, const float* uniforms, int ld_u,
                                    uint32_t* seen, int* codes, int ld_codes, int* finished, TtbArState* state,
                                    const TtbSampleParams* params, int stop_token, int advance, const int* row_start,
                                    void* stream) {
  const size_t smem = (size_t)V * sizeof(float);
  if (smem > 40 * 1024) { set_error("ttb_ar_sample_params: vocabulary %d too large", V); return -1; }
  if (!params) { set_error("ttb_ar_sample_params: params is NULL"); return -1; }
  if (row_start && (ld_codes <= 0 || ld_u <= 0)) {
    set_error("ttb_ar_sample_params: row_start needs ld_codes, ld_u > 0");
    return -1;
  }
  ar_sample_params_kernel<<<B, SAMP_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(
      logits, ld_logits, V, uniforms, ld_u, seen, codes, ld_codes, finished, state, params, stop_token, advance ? 1 : 0,
      row_start);
  TTB_CHECK_LAUNCH("ar_sample_params_kernel");
  return 0;
}

extern "C" int ttb_ar_fix_codes(int* codes, int B, int L, int stop_token, int* trim_len, void* stream) {
  ar_fix_codes_kernel<<<(B + 63) / 64, 64, 0, static_cast<cudaStream_t>(stream)>>>(codes, B, L, stop_token, trim_len);
  TTB_CHECK_LAUNCH("ar_fix_codes_kernel");
  return 0;
}
