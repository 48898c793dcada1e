// wav2vec2 CTC aligner kernels (prompt redaction, utils/wav2vec_alignment.py:58-123): the parts of Wav2Vec2ForCTC's
// forward that are not a GEMM, a LayerNorm over hidden states or attention (those run on ttb_gemm / ttb_layernorm /
// ttb_attention).
//   * ttb_wav2vec_conv0   = clip normalisation (wav2vec_alignment.py:65) + feature-extractor conv layer 0 (1 -> C,
//                           k = 10, stride 5, bias) + LayerNorm over the C channels + exact GELU (HF
//                           Wav2Vec2LayerNormConvLayer), token-major bf16 out
//   * ttb_layernorm_act   = LayerNorm over fp32 rows + optional exact GELU (conv layers 1-6 after their GEMM)
//   * ttb_argmax_rows     = logits.argmax(-1) (wav2vec_alignment.py:70,97)
#include "common.cuh"
#include "ttb_internal.h"

namespace ttb {

constexpr int W2V_STATS_THREADS = 1024;
constexpr int W2V_CONV0_K = 10, W2V_CONV0_S = 5;
constexpr int W2V_CONV0_MAXC = 512;

// Mean and unbiased standard deviation of the whole clip, one CTA, float64 partial sums in a fixed tree (no atomics:
// the same clip gives the same bits). stats[0] = mean, stats[1] = sqrt(var + 1e-7).
__global__ void __launch_bounds__(W2V_STATS_THREADS) w2v_clip_stats_kernel(const float* __restrict__ x, int n,
                                                                            float* __restrict__ stats) {
  __shared__ double red[W2V_STATS_THREADS / 32];
  __shared__ double bc;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  double s = 0.0;
  for (int i = threadIdx.x; i < n; i += W2V_STATS_THREADS) s += (double)x[i];
  for (int pass = 0; pass < 2; ++pass) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) red[w] = s;
    __syncthreads();
    if (w == 0) {
      double r = lane < W2V_STATS_THREADS / 32 ? red[lane] : 0.0;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
      if (lane == 0) bc = r;
    }
    __syncthreads();
    if (pass == 0) {
      const double mean = bc / n;
      if (threadIdx.x == 0) stats[0] = (float)mean;
      s = 0.0;
      for (int i = threadIdx.x; i < n; i += W2V_STATS_THREADS) {
        const double d = (double)x[i] - mean;
        s += d * d;
      }
      __syncthreads();           // red / bc are reused by the second pass
    } else if (threadIdx.x == 0) {
      stats[1] = sqrtf((float)(bc / (n - 1)) + 1e-7f);
    }
  }
}

// One warp per output frame t (samples 5t .. 5t+9 of the normalised clip); lane l owns channels l, l + 32, ...
// Weights live transposed in shared memory ([k][c]: the 32 lanes read 32 consecutive words).
__global__ void __launch_bounds__(256) w2v_conv0_kernel(const float* __restrict__ x, int n, const float* __restrict__ stats,
                                                        const float* __restrict__ w, const float* __restrict__ b,
                                                        const float* __restrict__ g, const float* __restrict__ beta, int C,
                                                        int L0, __nv_bfloat16* __restrict__ out, int ldo) {
  __shared__ float wt[W2V_CONV0_K * W2V_CONV0_MAXC];
  __shared__ float sb[W2V_CONV0_MAXC], sg[W2V_CONV0_MAXC], sbeta[W2V_CONV0_MAXC];
  for (int i = threadIdx.x; i < C * W2V_CONV0_K; i += blockDim.x) {
    const int c = i / W2V_CONV0_K, k = i - c * W2V_CONV0_K;
    wt[k * C + c] = w[i];
  }
  for (int c = threadIdx.x; c < C; c += blockDim.x) { sb[c] = b[c]; sg[c] = g[c]; sbeta[c] = beta[c]; }
  __syncthreads();
  const float mean = stats[0], sd = stats[1];
  const int lane = threadIdx.x & 31;
  const int nv = C >> 5;
  const float inv_c = 1.0f / (float)C;
  for (int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); t < L0; t += gridDim.x * (blockDim.x >> 5)) {
    const float xs = lane < W2V_CONV0_K ? (x[t * W2V_CONV0_S + lane] - mean) / sd : 0.f;
    float xk[W2V_CONV0_K];
#pragma unroll
    for (int k = 0; k < W2V_CONV0_K; ++k) xk[k] = __shfl_sync(0xffffffffu, xs, k);
    float v[W2V_CONV0_MAXC / 32];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < W2V_CONV0_MAXC / 32; ++i) {
      v[i] = 0.f;
      if (i < nv) {
        const int c = lane + 32 * i;
        float acc = sb[c];
#pragma unroll
        for (int k = 0; k < W2V_CONV0_K; ++k) acc = fmaf(wt[k * C + c], xk[k], acc);
        v[i] = acc;
        s += acc;
      }
    }
    const float mu = warp_sum(s) * inv_c;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < W2V_CONV0_MAXC / 32; ++i)
      if (i < nv) { const float d = v[i] - mu; q += d * d; }
    const float rstd = rsqrtf(warp_sum(q) * inv_c + 1e-5f);
    __nv_bfloat16* orow = out + (long long)t * ldo;
#pragma unroll
    for (int i = 0; i < W2V_CONV0_MAXC / 32; ++i)
      if (i < nv) {
        const int c = lane + 32 * i;
        orow[c] = __float2bfloat16(gelu_erf(fmaf((v[i] - mu) * rstd, sg[c], sbeta[c])));
      }
  }
}

// One warp per row of D = 128 * NV fp32 values (NV float4 per lane): two-pass statistics, eps 1e-5 as nn.LayerNorm.
template <int NV>
__global__ void __launch_bounds__(128) w2v_layernorm_act_kernel(const float* __restrict__ x, int M, int D,
                                                                const float* __restrict__ g, const float* __restrict__ b,
                                                                int gelu, __nv_bfloat16* __restrict__ ob,
                                                                float* __restrict__ of) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * 4 + (threadIdx.x >> 5);
  if (row >= M) return;
  const float* xr = x + row * D;
  float4 v[NV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    v[i] = *reinterpret_cast<const float4*>(xr + (i * 32 + lane) * 4);
    s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  }
  const float mean = warp_sum(s) / D;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float a = v[i].x - mean, bb = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    q += (a * a + bb * bb) + (c * c + d * d);
  }
  const float rstd = rsqrtf(warp_sum(q) / D + 1e-5f);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = (i * 32 + lane) * 4;
    const float4 gg = *reinterpret_cast<const float4*>(g + c), bq = *reinterpret_cast<const float4*>(b + c);
    float4 y;
    y.x = fmaf((v[i].x - mean) * rstd, gg.x, bq.x);
    y.y = fmaf((v[i].y - mean) * rstd, gg.y, bq.y);
    y.z = fmaf((v[i].z - mean) * rstd, gg.z, bq.z);
    y.w = fmaf((v[i].w - mean) * rstd, gg.w, bq.w);
    if (gelu) { y.x = gelu_erf(y.x); y.y = gelu_erf(y.y); y.z = gelu_erf(y.z); y.w = gelu_erf(y.w); }
    if (of) *reinterpret_cast<float4*>(of + row * D + c) = y;
    if (ob) *reinterpret_cast<uint2*>(ob + row * D + c) = make_uint2(pack_bf16(y.x, y.y), pack_bf16(y.z, y.w));
  }
}

// (value, index) order of torch.argmax: larger value wins, NaN beats every number, equal values -> smaller index.
TTB_DEVINL bool argmax_better(float v, int i, float bv, int bi) {
  const bool vn = isnan(v), bn = isnan(bv);
  if (vn != bn) return vn;
  if (!vn && v != bv) return v > bv;
  return i < bi;
}

// One warp per row.
__global__ void __launch_bounds__(128) argmax_rows_kernel(const float* __restrict__ x, int T, int V, int* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * 4 + (threadIdx.x >> 5);
  if (row >= T) return;
  const float* xr = x + row * V;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int j = lane; j < V; j += 32) {
    const float v = xr[j];
    if (argmax_better(v, j, best, bi)) { best = v; bi = j; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (argmax_better(ov, oi, best, bi)) { best = ov; bi = oi; }
  }
  if (lane == 0) out[row] = bi;
}

}  // namespace ttb

using namespace ttb;

extern "C" int ttb_wav2vec_conv0(const float* x, int n, const float* w, const float* b, const float* g, const float* beta,
                                 int C, float* stats, void* out_bf16, int ldo, void* stream) {
  if (n < W2V_CONV0_K || C <= 0 || C > W2V_CONV0_MAXC || (C & 31) || ldo < C || !x || !w || !b || !g || !beta || !stats ||
      !out_bf16) {
    set_error("ttb_wav2vec_conv0: bad arguments (n=%d >= 10, C=%d a multiple of 32 <= 512, ldo=%d >= C)", n, C, ldo);
    return -1;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int L0 = (n - W2V_CONV0_K) / W2V_CONV0_S + 1;
  w2v_clip_stats_kernel<<<1, W2V_STATS_THREADS, 0, st>>>(x, n, stats);
  TTB_CHECK_LAUNCH("w2v_clip_stats_kernel");
  const int blocks = (L0 + 7) / 8 < 132 * 8 ? (L0 + 7) / 8 : 132 * 8;
  w2v_conv0_kernel<<<blocks, 256, 0, st>>>(x, n, stats, w, b, g, beta, C, L0, reinterpret_cast<__nv_bfloat16*>(out_bf16), ldo);
  TTB_CHECK_LAUNCH("w2v_conv0_kernel");
  return 0;
}

extern "C" int ttb_layernorm_act(const float* x, int M, int D, const float* g, const float* b, int gelu, void* out_bf16,
                                 float* out_f32, void* stream) {
  if (M <= 0 || D <= 0 || (D & 127) || D > 1024 || !x || !g || !b || (!out_bf16 && !out_f32)) {
    set_error("ttb_layernorm_act: bad arguments (M=%d, D=%d must be a multiple of 128 <= 1024, one output)", M, D);
    return -1;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  __nv_bfloat16* ob = reinterpret_cast<__nv_bfloat16*>(out_bf16);
  const dim3 grid((M + 3) / 4);
  switch (D / 128) {
    case 1: w2v_layernorm_act_kernel<1><<<grid, 128, 0, st>>>(x, M, D, g, b, gelu, ob, out_f32); break;
    case 2: w2v_layernorm_act_kernel<2><<<grid, 128, 0, st>>>(x, M, D, g, b, gelu, ob, out_f32); break;
    case 3: w2v_layernorm_act_kernel<3><<<grid, 128, 0, st>>>(x, M, D, g, b, gelu, ob, out_f32); break;
    case 4: w2v_layernorm_act_kernel<4><<<grid, 128, 0, st>>>(x, M, D, g, b, gelu, ob, out_f32); break;
    case 5: w2v_layernorm_act_kernel<5><<<grid, 128, 0, st>>>(x, M, D, g, b, gelu, ob, out_f32); break;
    case 6: w2v_layernorm_act_kernel<6><<<grid, 128, 0, st>>>(x, M, D, g, b, gelu, ob, out_f32); break;
    case 7: w2v_layernorm_act_kernel<7><<<grid, 128, 0, st>>>(x, M, D, g, b, gelu, ob, out_f32); break;
    default: w2v_layernorm_act_kernel<8><<<grid, 128, 0, st>>>(x, M, D, g, b, gelu, ob, out_f32); break;
  }
  TTB_CHECK_LAUNCH("w2v_layernorm_act_kernel");
  return 0;
}

extern "C" int ttb_argmax_rows(const float* x, int T, int V, int* out, void* stream) {
  if (T <= 0 || V <= 0 || !x || !out) { set_error("ttb_argmax_rows: bad arguments (T=%d, V=%d)", T, V); return -1; }
  argmax_rows_kernel<<<(T + 3) / 4, 128, 0, static_cast<cudaStream_t>(stream)>>>(x, T, V, out);
  TTB_CHECK_LAUNCH("argmax_rows_kernel");
  return 0;
}
