// CLVP helpers (rotary, pooled LayerNorm, latent projection/score), diffusion helpers (timestep embedding, small
// fp32 linears, nearest interpolation, the fused DDPM step epilogue) and small layout utilities.
#include "common.cuh"
#include <cstring>
#include "ttb_internal.h"

namespace ttb {

// ------------------------------------------------------------------ CLVP rotary on q, k, v (first 32 dims / head)
// qkv bf16 [nseq*T, 3*H*64]; thread per (token, which in {q,k,v}, head, pair i in [0,16))
__global__ void clvp_rotary_kernel(__nv_bfloat16* __restrict__ qkv, int nseq, int T, int H) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)nseq * T * 3 * H * 16;
  if (idx >= total) return;
  const int i = (int)(idx & 15);
  long long r = idx >> 4;
  const int hh = (int)(r % (3 * H));       // which*H + head  (columns are [q heads | k heads | v heads])
  const long long tok = r / (3 * H);
  const int t = (int)(tok % T);
  // inv_freq_i = 10000^(-2i/32); angle = t * inv_freq_i; pairs (i, i+16) rotate (rotate_half, xtransformers.py:274-283)
  const float inv_freq = __powf(10000.0f, -(float)(2 * i) / 32.0f);
  const float ang = (float)t * inv_freq;
  float sn, cs;
  sincosf(ang, &sn, &cs);
  __nv_bfloat16* p = qkv + tok * (3LL * H * 64) + (long long)hh * 64;
  const float x1 = __bfloat162float(p[i]), x2 = __bfloat162float(p[i + 16]);
  p[i] = __float2bfloat16(x1 * cs - x2 * sn);
  p[i + 16] = __float2bfloat16(x2 * cs + x1 * sn);
}

// LayerNorm per token then mean over T tokens. grid (nseq), block 256 (8 warps, warp per token).
__global__ void __launch_bounds__(256)
clvp_pool_kernel(const float* __restrict__ x, int T, int D, const float* __restrict__ g, const float* __restrict__ b,
                 float* __restrict__ out) {
  extern __shared__ float acc[];  // [8][D]
  const int seq = blockIdx.x;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int c = lane; c < D; c += 32) acc[w * D + c] = 0.f;
  for (int t = w; t < T; t += 8) {
    const float* xr = x + ((long long)seq * T + t) * D;
    float s = 0.f;
    for (int c = lane; c < D; c += 32) s += xr[c];
    const float mean = warp_sum(s) / D;
    float q = 0.f;
    for (int c = lane; c < D; c += 32) { float d = xr[c] - mean; q += d * d; }
    const float rstd = rsqrtf(warp_sum(q) / D + 1e-5f);
    for (int c = lane; c < D; c += 32) acc[w * D + c] += (xr[c] - mean) * rstd * g[c] + b[c];
  }
  __syncthreads();
  for (int c = threadIdx.x; c < D; c += 256) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += acc[i * D + c];
    out[(long long)seq * D + c] = s / T;
  }
}

// latent = normalize(pooled @ W^T); optional score. grid (n), block 256; W fp32 [D, D] row-major (out, in)
__global__ void __launch_bounds__(256)
clvp_project_kernel(const float* __restrict__ pooled, int D, const float* __restrict__ W, float* __restrict__ latents,
                    const float* __restrict__ text_latent, float temp_exp, float* __restrict__ scores) {
  extern __shared__ float sh[];  // pooled row [D] + out [D]
  __shared__ float red[32];
  float* xin = sh;
  float* y = sh + D;
  const int r = blockIdx.x;
  for (int c = threadIdx.x; c < D; c += 256) xin[c] = pooled[(long long)r * D + c];
  __syncthreads();
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int o = w; o < D; o += 8) {
    const float* wr = W + (long long)o * D;
    float s = 0.f;
    for (int c = lane; c < D; c += 32) s += wr[c] * xin[c];
    s = warp_sum(s);
    if (lane == 0) y[o] = s;
  }
  __syncthreads();
  float q = 0.f;
  for (int c = threadIdx.x; c < D; c += 256) q += y[c] * y[c];
  const float nrm = fmaxf(sqrtf(block_sum(q, red)), 1e-12f);   // F.normalize eps
  float dot = 0.f;
  for (int c = threadIdx.x; c < D; c += 256) {
    const float v = y[c] / nrm;
    if (latents) latents[(long long)r * D + c] = v;
    if (text_latent) dot += v * text_latent[c];
  }
  if (text_latent) {
    dot = block_sum(dot, red);
    if (threadIdx.x == 0) scores[r] = dot * temp_exp;
  }
}

// ------------------------------------------------------------------ diffusion helpers
__global__ void timestep_embedding_kernel(const int* __restrict__ t, int C, float* __restrict__ out) {
  const int r = blockIdx.x;
  const int half = C / 2;
  const float tv = (float)t[r];
  for (int i = threadIdx.x; i < half; i += blockDim.x) {
    const float f = expf(-logf(10000.0f) * (float)i / (float)half);
    const float a = tv * f;
    out[(long long)r * C + i] = cosf(a);
    out[(long long)r * C + half + i] = sinf(a);
  }
}

// out[m, n] = act_out( sum_k act_in(x[m,k]) W[n,k] + b[n] ); warp per output, fp32 (M is tiny: timesteps)
__global__ void __launch_bounds__(256)
linear_small_kernel(const float* __restrict__ x, int M, int K, const float* __restrict__ W, const float* __restrict__ b,
                    int N, int silu_in, int silu_out, float* __restrict__ out) {
  extern __shared__ float xs[];  // K
  const int m = blockIdx.y;
  for (int k = threadIdx.x; k < K; k += 256) { float v = x[(long long)m * K + k]; xs[k] = silu_in ? silu(v) : v; }
  __syncthreads();
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = blockIdx.x * 8 + w;
  if (n >= N) return;
  const float* wr = W + (long long)n * K;
  float s = 0.f;
  for (int k = lane; k < K; k += 32) s += wr[k] * xs[k];
  s = warp_sum(s);
  if (lane == 0) {
    s += b ? b[n] : 0.f;
    out[(long long)m * N + n] = silu_out ? silu(s) : s;
  }
}

__global__ void interp_nearest_kernel(const float* __restrict__ x, int N, int S, int C, __nv_bfloat16* __restrict__ ob,
                                      int ldo, float* __restrict__ of, int ldof) {
  const int s = blockIdx.x;
  // PyTorch 'nearest': src = floor(dst * (N / S)) computed in float: scale = (float)N / S
  const float scale = (float)N / (float)S;
  int src = (int)floorf((float)s * scale);
  src = min(src, N - 1);
  const float* xr = x + (long long)src * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float v = xr[c];
    if (ob) ob[(long long)s * ldo + c] = __float2bfloat16(v);
    if (of) of[(long long)s * ldof + c] = v;
  }
}

// DDPM step epilogue. One thread per (s, c).
__global__ void __launch_bounds__(256)
diffusion_step_kernel(TtbDiffStepArgs a) {
  const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
  if (idx >= (long long)a.S * a.C) return;
  const int s = (int)(idx / a.C), c = (int)(idx - (long long)s * a.C);
  const int call = *a.step;
  const int i = a.iters - 1 - call;
  const float* tb = a.tables;
  const float sra = tb[0 * a.iters + i], srm1 = tb[1 * a.iters + i], minlog = tb[2 * a.iters + i],
              maxlog = tb[3 * a.iters + i], c1 = tb[4 * a.iters + i], c2 = tb[5 * a.iters + i];
  // parity_stride != 0: the two CFG branches arrive through the double-buffered peer-exchange area (ttb_pair_exchange)
  const float* mob = a.model_out + (long long)(call & 1) * a.parity_stride;
  const float* mo = mob + (long long)s * a.ld_out;
  float eps = mo[c];
  const float var = mo[a.C + c];
  if (a.cond_free) {
    const float eps_u = mob[a.out_bstride + (long long)s * a.ld_out + c];
    // cfk = k * (1 - i / iters)  (utils/diffusion.py:377-383), computed in double as Python does, then fp32 math
    const double cfkd = (double)a.cond_free_k * (1.0 - (double)i / (double)a.iters);
    eps = (float)(1.0 + cfkd) * eps - (float)cfkd * eps_u;
  }
  const float frac = (var + 1.0f) / 2.0f;
  const float logvar = frac * maxlog + (1.0f - frac) * minlog;
  const float xt = a.x[idx];
  float x0 = sra * xt - srm1 * eps;
  x0 = fminf(fmaxf(x0, -1.0f), 1.0f);
  const float mean = c1 * x0 + c2 * xt;
  const float nz = (i == 0) ? 0.f : 1.f;
  const float noise = a.noise[(long long)call * a.S * a.C + idx];
  const float xn = mean + nz * expf(0.5f * logvar) * noise;
  a.x[idx] = xn;
  if (a.x_bf16) reinterpret_cast<__nv_bfloat16*>(a.x_bf16)[(long long)s * a.ld_xb + c] = __float2bfloat16(xn);
  if (a.mel_out && i == 0) {
    const float MX = 2.3143386840820312f, MN = -11.512925148010254f;
    a.mel_out[(long long)c * a.S + s] = ((xn + 1.0f) / 2.0f) * (MX - MN) + MN;
  }
}

// DDIM step epilogue (eq. 12 of Song et al.). One thread per (s, c). The learned-variance half of model_out is not read.
__global__ void __launch_bounds__(256)
ddim_step_kernel(TtbDiffStepArgs a) {
  const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
  if (idx >= (long long)a.S * a.C) return;
  const int s = (int)(idx / a.C), c = (int)(idx - (long long)s * a.C);
  const int call = *a.step;
  const int i = a.iters - 1 - call;
  const float* tb = a.tables;
  const float sra = tb[0 * a.iters + i], srm1 = tb[1 * a.iters + i], sab_prev = tb[2 * a.iters + i],
              dir = tb[3 * a.iters + i], sigma = tb[4 * a.iters + i];
  const float* mob = a.model_out + (long long)(call & 1) * a.parity_stride;
  float eps = mob[(long long)s * a.ld_out + c];
  if (a.cond_free) {
    const float eps_u = mob[a.out_bstride + (long long)s * a.ld_out + c];
    const double cfkd = (double)a.cond_free_k * (1.0 - (double)i / (double)a.iters);
    eps = (float)(1.0 + cfkd) * eps - (float)cfkd * eps_u;
  }
  const float xt = a.x[idx];
  const float sx = sra * xt;
  const float x0 = fminf(fmaxf(sx - srm1 * eps, -1.0f), 1.0f);
  // eps re-derived from the clamped x0 (_predict_eps_from_xstart), not the model's eps
  const float eps_x0 = (sx - x0) / srm1;
  const float nz = (i == 0) ? 0.f : 1.f;
  const float noise = a.noise ? a.noise[(long long)call * a.S * a.C + idx] : 0.f;
  const float xn = (sab_prev * x0 + dir * eps_x0) + nz * sigma * noise;
  a.x[idx] = xn;
  if (a.x_bf16) reinterpret_cast<__nv_bfloat16*>(a.x_bf16)[(long long)s * a.ld_xb + c] = __float2bfloat16(xn);
  if (a.mel_out && i == 0) {
    const float MX = 2.3143386840820312f, MN = -11.512925148010254f;
    a.mel_out[(long long)c * a.S + s] = ((xn + 1.0f) / 2.0f) * (MX - MN) + MN;
  }
}

// DPM-Solver++(2M) step epilogue (Lu et al. 2022, Algorithm 2). One thread per (s, c). The learned-variance half of
// model_out is not read. x0_prev [S, C] carries the clamped x0 of the previous call.
__global__ void __launch_bounds__(256)
dpmpp2m_step_kernel(TtbDiffStepArgs a, float* __restrict__ x0_prev) {
  const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
  if (idx >= (long long)a.S * a.C) return;
  const int s = (int)(idx / a.C), c = (int)(idx - (long long)s * a.C);
  const int call = *a.step;
  const int i = a.iters - 1 - call;
  const float* tb = a.tables;
  const float sra = tb[0 * a.iters + i], srm1 = tb[1 * a.iters + i], ca = tb[2 * a.iters + i], cb = tb[3 * a.iters + i],
              w = tb[4 * a.iters + i], wp = tb[5 * a.iters + i];
  const float* mob = a.model_out + (long long)(call & 1) * a.parity_stride;
  float eps = mob[(long long)s * a.ld_out + c];
  if (a.cond_free) {
    const float eps_u = mob[a.out_bstride + (long long)s * a.ld_out + c];
    const double cfkd = (double)a.cond_free_k * (1.0 - (double)i / (double)a.iters);
    eps = (float)(1.0 + cfkd) * eps - (float)cfkd * eps_u;
  }
  const float xt = a.x[idx];
  const float d = fminf(fmaxf(sra * xt - srm1 * eps, -1.0f), 1.0f);
  // a first-order step (wp == 0: first and last call) does not read x0_prev, which holds nothing of this chain yet
  const float dm = (wp != 0.f) ? w * d + wp * x0_prev[idx] : w * d;
  const float xn = ca * xt + cb * dm;
  x0_prev[idx] = d;
  a.x[idx] = xn;
  if (a.x_bf16) reinterpret_cast<__nv_bfloat16*>(a.x_bf16)[(long long)s * a.ld_xb + c] = __float2bfloat16(xn);
  if (a.mel_out && i == 0) {
    const float MX = 2.3143386840820312f, MN = -11.512925148010254f;
    a.mel_out[(long long)c * a.S + s] = ((xn + 1.0f) / 2.0f) * (MX - MN) + MN;
  }
}

__global__ void counter_add_kernel(int* c, int d) { *c += d; }

// ------------------------------------------------------------------ CFG pair: exchange of the two denoiser branches
// Two GPUs evaluate one classifier-free-guidance branch each (diffusion_engine.py). The fallback exchanges the [S, 200] fp32
// outputs with an eager NCCL all-gather between two CUDA graphs per step, which costs more than the step's compute.
// This kernel is the exchange as ONE graph-capturable launch over peer memory (CUDA IPC mapping of the partner's buffer,
// NVLink stores): copy my branch into slot (step parity, my branch) of BOTH exchange areas, publish a flag in the
// partner's memory, wait for the partner's flag. Slots are double-buffered by step parity: the partner can be at most one
// step ahead (it needs my data of its current step), so it never overwrites a slot I still read.
__global__ void __launch_bounds__(256)
pair_exchange_kernel(const float4* __restrict__ src, float4* __restrict__ local_area, float4* __restrict__ peer_area,
                     long long n4, long long parity_stride4, long long branch_off4, int* peer_flags, int* my_flags,
                     const int* __restrict__ counter, const int* __restrict__ epoch, unsigned int* done_ctr, int* err) {
  const int call = *counter;
  const int want = *epoch + call + 1;
  const long long off = (long long)(call & 1) * parity_stride4 + branch_off4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = src[i];
    local_area[off + i] = v;
    peer_area[off + i] = v;
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int t = atomicAdd(done_ctr, 1u);
    if (t == gridDim.x - 1) {                       // last CTA: every store of this launch is visible system-wide
      *done_ctr = 0;
      asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(peer_flags + (call & 1)), "r"(want) : "memory");
      const unsigned long long t0 = global_timer_ns();
      int seen;
      do {
        asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(seen) : "l"(my_flags + (call & 1)) : "memory");
        if (seen - want < 0 && global_timer_ns() - t0 > 5000000000ull) { *err = 1; break; }   // 5 s: partner is gone
      } while (seen - want < 0);
    }
  }
}

__global__ void transpose_f32_kernel(const float* __restrict__ in, int R, int C, float* __restrict__ out) {
  __shared__ float tile[32][33];
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int r = r0 + i, c = c0 + threadIdx.x;
    if (r < R && c < C) tile[i][threadIdx.x] = in[(long long)r * C + c];
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int c = c0 + i, r = r0 + threadIdx.x;
    if (r < R && c < C) out[(long long)c * R + r] = tile[threadIdx.x][i];
  }
}

__global__ void cast_pad_bf16_kernel(const float* __restrict__ in, int R, int C, int ld_in, __nv_bfloat16* __restrict__ out,
                                     int ldo, int ncols) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)R * ncols) return;
  const int r = (int)(idx / ncols), c = (int)(idx - (long long)r * ncols);
  out[(long long)r * ldo + c] = __float2bfloat16(c < C ? in[(long long)r * ld_in + c] : 0.f);
}

__global__ void broadcast_rows_kernel(const float* __restrict__ row, int R, int C, float* __restrict__ of,
                                      __nv_bfloat16* __restrict__ ob, int ldo) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)R * C) return;
  const int r = (int)(idx / C), c = (int)(idx - (long long)r * C);
  if (of) of[(long long)r * ldo + c] = row[c];
  if (ob) ob[(long long)r * ldo + c] = __float2bfloat16(row[c]);
}

}  // namespace ttb
using namespace ttb;
#define ST static_cast<cudaStream_t>(stream)

extern "C" int ttb_clvp_rotary(void* qkv, int nseq, int T, int H, void* stream) {
  const long long total = (long long)nseq * T * 3 * H * 16;
  if (total <= 0) return 0;
  clvp_rotary_kernel<<<(unsigned)((total + 255) / 256), 256, 0, ST>>>(reinterpret_cast<__nv_bfloat16*>(qkv), nseq, T, H);
  TTB_CHECK_LAUNCH("clvp_rotary_kernel");
  return 0;
}
extern "C" int ttb_clvp_pool(const float* x, int nseq, int T, int D, const float* g, const float* b, float* out, void* stream) {
  clvp_pool_kernel<<<nseq, 256, 8 * D * sizeof(float), ST>>>(x, T, D, g, b, out);
  TTB_CHECK_LAUNCH("clvp_pool_kernel");
  return 0;
}
extern "C" int ttb_clvp_project(const float* pooled, int n, int D, const float* W, float* latents, const float* text_latent,
                                float temp_exp, float* scores, void* stream) {
  clvp_project_kernel<<<n, 256, 2 * D * sizeof(float), ST>>>(pooled, D, W, latents, text_latent, temp_exp, scores);
  TTB_CHECK_LAUNCH("clvp_project_kernel");
  return 0;
}
extern "C" int ttb_timestep_embedding(const int* t, int n, int C, float* out, void* stream) {
  timestep_embedding_kernel<<<n, 256, 0, ST>>>(t, C, out);
  TTB_CHECK_LAUNCH("timestep_embedding_kernel");
  return 0;
}
extern "C" int ttb_linear_small(const float* x, int M, int K, const float* W, const float* b, int N, int silu_in,
                                int silu_out, float* out, void* stream) {
  dim3 grid((N + 7) / 8, M);
  linear_small_kernel<<<grid, 256, K * sizeof(float), ST>>>(x, M, K, W, b, N, silu_in, silu_out, out);
  TTB_CHECK_LAUNCH("linear_small_kernel");
  return 0;
}
extern "C" int ttb_interp_nearest(const float* x, int N, int S, int C, void* out_bf16, int ldo, float* out_f32, int ldof,
                                  void* stream) {
  interp_nearest_kernel<<<S, 256, 0, ST>>>(x, N, S, C, reinterpret_cast<__nv_bfloat16*>(out_bf16), ldo, out_f32, ldof);
  TTB_CHECK_LAUNCH("interp_nearest_kernel");
  return 0;
}
extern "C" int ttb_diffusion_step(const TtbDiffStepArgs* args, void* stream) {
  const long long n = (long long)args->S * args->C;
  diffusion_step_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ST>>>(*args);
  TTB_CHECK_LAUNCH("diffusion_step_kernel");
  return 0;
}
extern "C" int ttb_ddim_step(const TtbDiffStepArgs* args, void* stream) {
  const long long n = (long long)args->S * args->C;
  ddim_step_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ST>>>(*args);
  TTB_CHECK_LAUNCH("ddim_step_kernel");
  return 0;
}
extern "C" int ttb_dpmpp2m_step(const TtbDiffStepArgs* args, float* x0_prev, void* stream) {
  if (!x0_prev) { set_error("ttb_dpmpp2m_step: x0_prev is required"); return -1; }
  const long long n = (long long)args->S * args->C;
  dpmpp2m_step_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ST>>>(*args, x0_prev);
  TTB_CHECK_LAUNCH("dpmpp2m_step_kernel");
  return 0;
}
extern "C" int ttb_pair_exchange(const float* src, float* local_area, float* peer_area, long long n, long long parity_stride,
                                 long long branch_off, int* peer_flags, int* my_flags, const int* counter, const int* epoch,
                                 unsigned int* done_ctr, int* err, void* stream) {
  if ((n & 3) || (parity_stride & 3) || (branch_off & 3)) { set_error("ttb_pair_exchange: sizes must be multiples of 4 floats"); return -1; }
  pair_exchange_kernel<<<64, 256, 0, ST>>>(reinterpret_cast<const float4*>(src), reinterpret_cast<float4*>(local_area),
                                           reinterpret_cast<float4*>(peer_area), n / 4, parity_stride / 4, branch_off / 4,
                                           peer_flags, my_flags, counter, epoch, done_ctr, err);
  TTB_CHECK_LAUNCH("pair_exchange_kernel");
  return 0;
}
// Exchange buffers live in their own cudaMalloc allocations (not in a caching allocator's pool) so that the IPC handle
// describes exactly the buffer; the partner opens it with its OWN device current, which lets the driver enable peer
// access between the two devices for that mapping (cudaIpcMemLazyEnablePeerAccess).
extern "C" int ttb_peer_alloc(long long bytes, void** ptr, void* handle64) {
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, (size_t)bytes);
  if (e == cudaSuccess) e = cudaMemset(p, 0, (size_t)bytes);
  cudaIpcMemHandle_t h;
  if (e == cudaSuccess) e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) { if (p) cudaFree(p); return check_cuda(e, "ttb_peer_alloc"); }
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  memcpy(handle64, &h, 64);
  *ptr = p;
  return 0;
}
extern "C" int ttb_peer_open(const void* handle64, void** ptr) {
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  void* p = nullptr;
  const cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) return check_cuda(e, "cudaIpcOpenMemHandle");
  *ptr = p;
  return 0;
}
extern "C" int ttb_peer_close(void* ptr) { return check_cuda(cudaIpcCloseMemHandle(ptr), "cudaIpcCloseMemHandle"); }
extern "C" int ttb_peer_free(void* ptr) { return check_cuda(cudaFree(ptr), "cudaFree"); }
extern "C" int ttb_enable_peer_access(int peer_device) {
  int dev = 0;
  cudaGetDevice(&dev);
  if (peer_device == dev) return 0;
  int can = 0;
  cudaDeviceCanAccessPeer(&can, dev, peer_device);
  if (!can) { set_error("ttb_enable_peer_access: device %d cannot access device %d", dev, peer_device); return -1; }
  const cudaError_t e = cudaDeviceEnablePeerAccess(peer_device, 0);
  if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return check_cuda(e, "cudaDeviceEnablePeerAccess");
  cudaGetLastError();
  return 0;
}
namespace ttb {
__global__ void act_split_cast_kernel(const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ c,
                                      float scale, float slope, int R, int C, __nv_bfloat16* __restrict__ out, int ldo) {
  pdl_wait();
  const int groups = ldo >> 2;                        // 4 output columns per thread
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)R * groups) return;
  const int r = (int)(i / groups), g = (int)(i - (long long)r * groups);
  const int col = g * 4;
  uint32_t w0 = 0u, w1 = 0u;
  if (col < 3 * C) {
    const int part = col / C, cc = col - part * C;    // C % 4 == 0: a group never straddles two parts
    const long long off = (long long)r * C + cc;
    float4 v = *reinterpret_cast<const float4*>(a + off);
    if (b) { const float4 t = *reinterpret_cast<const float4*>(b + off); v.x += t.x; v.y += t.y; v.z += t.z; v.w += t.w; }
    if (c) { const float4 t = *reinterpret_cast<const float4*>(c + off); v.x += t.x; v.y += t.y; v.z += t.z; v.w += t.w; }
    float x[4] = {v.x * scale, v.y * scale, v.z * scale, v.w * scale};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      x[k] = x[k] > 0.f ? x[k] : x[k] * slope;
      if (part == 1) x[k] -= __bfloat162float(__float2bfloat16(x[k]));      // lo = v - bf16(v)
    }
    w0 = pack_bf16(x[0], x[1]);
    w1 = pack_bf16(x[2], x[3]);
  }
  *reinterpret_cast<uint2*>(out + (long long)r * ldo + col) = make_uint2(w0, w1);
}

__global__ void interp_linear_kernel(const float* __restrict__ x, int N, int C, float rscale, int S, float* __restrict__ out) {
  pdl_wait();
  const int c4 = C >> 2;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)S * c4) return;
  const int s = (int)(i / c4), c = (int)(i - (long long)s * c4) * 4;
  // area_pixel_compute_source_index (align_corners = False, explicit scale): negative sources clamp to 0
  float src = ((float)s + 0.5f) * rscale - 0.5f;
  src = src < 0.f ? 0.f : src;
  int i0 = (int)src;
  i0 = i0 > N - 1 ? N - 1 : i0;
  const int i1 = i0 + (i0 < N - 1 ? 1 : 0);
  const float l1 = src - (float)i0, l0 = 1.f - l1;
  const float4 p = *reinterpret_cast<const float4*>(x + (long long)i0 * C + c);
  const float4 q = *reinterpret_cast<const float4*>(x + (long long)i1 * C + c);
  *reinterpret_cast<float4*>(out + (long long)s * C + c) = make_float4(l0 * p.x + l1 * q.x, l0 * p.y + l1 * q.y,
                                                                         l0 * p.z + l1 * q.z, l0 * p.w + l1 * q.w);
}
}  // namespace ttb

extern "C" int ttb_act_split_cast(const float* a, const float* b, const float* c, float scale, float slope, int R, int C,
                                  void* out, int ldo, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if ((C & 3) || (ldo & 3) || ldo < 3 * C || R <= 0) { set_error("ttb_act_split_cast: C=%d ldo=%d unsupported", C, ldo); return -1; }
  const long long n = (long long)R * (ldo >> 2);
  launch_pdl(act_split_cast_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), (size_t)0, st, a, b, c, scale, slope, R, C,
             reinterpret_cast<__nv_bfloat16*>(out), ldo);
  TTB_CHECK_LAUNCH("act_split_cast_kernel");
  return 0;
}

extern "C" int ttb_interp_linear(const float* x, int N, int C, float rscale, int S, float* out, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if ((C & 3) || N <= 0 || S <= 0) { set_error("ttb_interp_linear: bad shape"); return -1; }
  const long long n = (long long)S * (C >> 2);
  launch_pdl(interp_linear_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), (size_t)0, st, x, N, C, rscale, S, out);
  TTB_CHECK_LAUNCH("interp_linear_kernel");
  return 0;
}

extern "C" int ttb_counter_add(int* counter, int delta, void* stream) {
  counter_add_kernel<<<1, 1, 0, ST>>>(counter, delta);
  TTB_CHECK_LAUNCH("counter_add_kernel");
  return 0;
}
extern "C" int ttb_transpose_f32(const float* in, int R, int Cc, float* out, void* stream) {
  dim3 grid((Cc + 31) / 32, (R + 31) / 32), block(32, 8);
  transpose_f32_kernel<<<grid, block, 0, ST>>>(in, R, Cc, out);
  TTB_CHECK_LAUNCH("transpose_f32_kernel");
  return 0;
}
extern "C" int ttb_cast_pad_bf16(const float* in, int R, int Cc, int ld_in, void* out, int ldo, int ncols_out, void* stream) {
  const long long n = (long long)R * ncols_out;
  if (n <= 0) return 0;
  cast_pad_bf16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ST>>>(in, R, Cc, ld_in, reinterpret_cast<__nv_bfloat16*>(out), ldo, ncols_out);
  TTB_CHECK_LAUNCH("cast_pad_bf16_kernel");
  return 0;
}
extern "C" int ttb_broadcast_rows(const float* row, int R, int Cc, float* out_f32, void* out_bf16, int ldo, void* stream) {
  const long long n = (long long)R * Cc;
  broadcast_rows_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ST>>>(row, R, Cc, out_f32, reinterpret_cast<__nv_bfloat16*>(out_bf16), ldo);
  TTB_CHECK_LAUNCH("broadcast_rows_kernel");
  return 0;
}
