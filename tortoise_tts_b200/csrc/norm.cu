// Normalisation kernels (HBM/L2-bound): LayerNorm (single or chained), RMSNorm, GroupNorm32 with the fused
// scale-shift / SiLU consumers. fp32 statistics via warp-shuffle reductions; outputs feed the wgmma GEMM as bf16.
#include "common.cuh"
#include "ttb_internal.h"

namespace ttb {

// one block (256 threads) per row; D <= 4096; row cached in registers (up to 16 per thread)
template <int MAXV>
__global__ void __launch_bounds__(256)
layernorm_kernel(const float* x, int D, const float* __restrict__ g1, const float* __restrict__ b1,
                 const float* __restrict__ g2, const float* __restrict__ b2, __nv_bfloat16* __restrict__ ob,
                 float* __restrict__ of, float* xw, const float* __restrict__ partials, int nsplit,
                 long long split_stride, const float* __restrict__ rbias) {
  __shared__ float red[32];
  const long long row = blockIdx.x;
  const float* xr = x + row * D;
  float v[MAXV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    int c = threadIdx.x + i * 256;
    v[i] = (c < D) ? xr[c] : 0.f;
    if (xw && c < D) {          // fused residual update: x += bias + sum of split-K partials (fixed order)
      float t = rbias ? rbias[c] : 0.f;
      for (int sp = 0; sp < nsplit; ++sp) t += partials[sp * split_stride + row * D + c];
      v[i] += t;
      xw[row * D + c] = v[i];
    }
    s += v[i];
  }
  float mean = block_sum(s, red) / D;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    int c = threadIdx.x + i * 256;
    float d = (c < D) ? v[i] - mean : 0.f;
    q += d * d;
  }
  float rstd = rsqrtf(block_sum(q, red) / D + 1e-5f);
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    int c = threadIdx.x + i * 256;
    if (c < D) v[i] = (v[i] - mean) * rstd * g1[c] + b1[c];
  }
  if (g2) {
    s = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) { int c = threadIdx.x + i * 256; s += (c < D) ? v[i] : 0.f; }
    mean = block_sum(s, red) / D;
    q = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      int c = threadIdx.x + i * 256;
      float d = (c < D) ? v[i] - mean : 0.f;
      q += d * d;
    }
    rstd = rsqrtf(block_sum(q, red) / D + 1e-5f);
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      int c = threadIdx.x + i * 256;
      if (c < D) v[i] = (v[i] - mean) * rstd * g2[c] + b2[c];
    }
  }
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    int c = threadIdx.x + i * 256;
    if (c < D) {
      if (ob) ob[row * D + c] = __float2bfloat16(v[i]);
      if (of) of[row * D + c] = v[i];
    }
  }
}

// One WARP per row (D = 128 * NV, NV <= 8): the row lives in NV float4 per lane, both statistics are xor-shuffle trees,
// no shared memory and no block barrier. The GPT-2 decode step runs 61 of these on 256 rows between skinny GEMMs
// (the two block_sum round trips of the block-per-row kernel above dominate a 4 KB row). Same arithmetic as layernorm_kernel (two-pass variance, fixed
// summation order of the split-K partials), only the reduction tree differs.

template <int NV>
__global__ void __launch_bounds__(64)
layernorm_warp_kernel(const float* x, int M, int D, const float* __restrict__ g1, const float* __restrict__ b1,
                      const float* __restrict__ g2, const float* __restrict__ b2, __nv_bfloat16* __restrict__ ob,
                      float* __restrict__ of, float* xw, const float* __restrict__ partials, int nsplit,
                      long long split_stride, const float* __restrict__ rbias, int early) {
  // `early`: let the next kernel's CTAs start NOW (TTB_LN_EARLY, default on). In the decode step that kernel is a
  // skinny GEMM with TtbGemmArgs.w_static: it runs its prologue and streams its weight tiles while this kernel works,
  // and still waits (griddepcontrol.wait) for this grid to finish before it touches the normalised rows. This kernel
  // needs no shared memory and few registers, so the early CTAs take nothing away from it.
  if (early) pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * 2 + (threadIdx.x >> 5);
  if (row >= M) return;
  const float* xr = x + row * D;
  float4 v[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = *reinterpret_cast<const float4*>(xr + (i * 32 + lane) * 4);
  if (xw) {                     // fused residual update: x += bias + sum of split-K partials (fixed order)
    float4 t[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i)
      t[i] = rbias ? *reinterpret_cast<const float4*>(rbias + (i * 32 + lane) * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
    for (int sp = 0; sp < nsplit; ++sp) {
      const float* pr = partials + sp * split_stride + row * D;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const float4 p = *reinterpret_cast<const float4*>(pr + (i * 32 + lane) * 4);
        t[i].x += p.x; t[i].y += p.y; t[i].z += p.z; t[i].w += p.w;
      }
    }
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      v[i].x += t[i].x; v[i].y += t[i].y; v[i].z += t[i].z; v[i].w += t[i].w;
      *reinterpret_cast<float4*>(xw + row * D + (i * 32 + lane) * 4) = v[i];
    }
  }
  if (!early) pdl_launch_dependents();        // tail trigger: every load of this row is done
#pragma unroll
  for (int pass = 0; pass < 2; ++pass) {
    const float* gg = pass == 0 ? g1 : g2;
    const float* bb = pass == 0 ? b1 : b2;
    if (!gg) break;
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    const float mean = warp_sum(s) / D;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const float dx = v[i].x - mean, dy = v[i].y - mean, dz = v[i].z - mean, dw = v[i].w - mean;
      q += (dx * dx + dy * dy) + (dz * dz + dw * dw);
    }
    const float rstd = rsqrtf(warp_sum(q) / D + 1e-5f);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const float4 ga = *reinterpret_cast<const float4*>(gg + (i * 32 + lane) * 4);
      const float4 be = *reinterpret_cast<const float4*>(bb + (i * 32 + lane) * 4);
      v[i].x = (v[i].x - mean) * rstd * ga.x + be.x;
      v[i].y = (v[i].y - mean) * rstd * ga.y + be.y;
      v[i].z = (v[i].z - mean) * rstd * ga.z + be.z;
      v[i].w = (v[i].w - mean) * rstd * ga.w + be.w;
    }
  }
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = (i * 32 + lane) * 4;
    if (ob) *reinterpret_cast<uint2*>(ob + row * D + c) = make_uint2(pack_bf16(v[i].x, v[i].y), pack_bf16(v[i].z, v[i].w));
    if (of) *reinterpret_cast<float4*>(of + row * D + c) = v[i];
  }
}

template <int MAXV>
__global__ void __launch_bounds__(256)
rmsnorm_kernel(const float* __restrict__ x, int D, const float* __restrict__ g, __nv_bfloat16* __restrict__ ob) {
  __shared__ float red[32];
  const long long row = blockIdx.x;
  const float* xr = x + row * D;
  float v[MAXV];
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    int c = threadIdx.x + i * 256;
    v[i] = (c < D) ? xr[c] : 0.f;
    q += v[i] * v[i];
  }
  float nrm = sqrtf(block_sum(q, red)) * rsqrtf((float)D);
  float inv = 1.0f / fmaxf(nrm, 1e-8f);
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    int c = threadIdx.x + i * 256;
    if (c < D) ob[row * D + c] = __float2bfloat16(v[i] * inv * g[c]);
  }
}

// GroupNorm statistics, token-major x [B, S, C]: grid (groups, splits, B); block 256 threads.
// Each block reduces rows [s0, s1) x channels of one group; partial (sum, sumsq) -> partials[b][g][split][2].
__global__ void __launch_bounds__(256)
gn_stats_kernel(const float* __restrict__ x, int S, int C, int cpg, int splits, float* __restrict__ partials) {
  __shared__ float red[32];
  const int g = blockIdx.x, sp = blockIdx.y, b = blockIdx.z;
  const int rows_per = (S + splits - 1) / splits;
  const int s0 = sp * rows_per, s1 = min(S, s0 + rows_per);
  const float* xb = x + (long long)b * S * C + g * cpg;
  float s = 0.f, q = 0.f;
  if ((cpg & 3) == 0) {
    const int vec = cpg >> 2;  // float4 per row
    const int total = (s1 - s0) * vec;
    for (int i = threadIdx.x; i < total; i += 256) {
      int r = i / vec, c = i - r * vec;
      float4 t = *reinterpret_cast<const float4*>(xb + (long long)(s0 + r) * C + c * 4);
      s += t.x + t.y + t.z + t.w;
      q += t.x * t.x + t.y * t.y + t.z * t.z + t.w * t.w;
    }
  } else {
    const int total = (s1 - s0) * cpg;
    for (int i = threadIdx.x; i < total; i += 256) {
      int r = i / cpg, c = i - r * cpg;
      float t = xb[(long long)(s0 + r) * C + c];
      s += t; q += t * t;
    }
  }
  s = block_sum(s, red);
  q = block_sum(q, red);
  if (threadIdx.x == 0) {
    float* p = partials + (((long long)b * gridDim.x + g) * splits + sp) * 2;
    p[0] = s; p[1] = q;
  }
}

// apply: each thread handles 4 consecutive channels of one token
__global__ void __launch_bounds__(256)
gn_apply_kernel(const float* __restrict__ x, int S, int C, int groups, int cpg, int splits,
                const float* __restrict__ partials, const float* __restrict__ gamma, const float* __restrict__ beta,
                const float* __restrict__ ss, int ss_bstride, const int* __restrict__ ss_row, int ss_row_stride,
                int do_silu, __nv_bfloat16* __restrict__ ob, int ldo,
                float* __restrict__ of, int ldof) {
  const int b = blockIdx.y;
  const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;  // over S * C/4
  const int c4 = C >> 2;
  if (idx >= (long long)S * c4) return;
  const int srow = (int)(idx / c4);
  const int c = (int)(idx - (long long)srow * c4) * 4;
  const int g = c / cpg;
  const float* p = partials + ((long long)b * groups + g) * splits * 2;
  float sum = 0.f, sq = 0.f;
  for (int i = 0; i < splits; ++i) { sum += p[2 * i]; sq += p[2 * i + 1]; }
  const float n = (float)S * cpg;
  const float mean = sum / n;
  const float var = fmaxf(sq / n - mean * mean, 0.f);
  const float rstd = rsqrtf(var + 1e-5f);
  if (ss && ss_row) ss += (long long)(*ss_row) * ss_row_stride;
  float4 t = *reinterpret_cast<const float4*>(x + ((long long)b * S + srow) * C + c);
  float v[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float y = (v[j] - mean) * rstd * gamma[c + j] + beta[c + j];
    if (ss) y = y * (1.0f + ss[(long long)b * ss_bstride + c + j]) + ss[(long long)b * ss_bstride + C + c + j];
    if (do_silu) y = silu(y);
    v[j] = y;
  }
  if (ob) {
    uint2 o = make_uint2(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]));
    *reinterpret_cast<uint2*>(ob + ((long long)b * S + srow) * ldo + c) = o;
  }
  if (of) *reinterpret_cast<float4*>(of + ((long long)b * S + srow) * ldof + c) = make_float4(v[0], v[1], v[2], v[3]);
}

// ---------------------------------------------------------------------------------------------------------------
// Row-wise GroupNorm (the path the denoiser takes: C = 1024, 32 groups). The two kernels above walk one GROUP at a
// time (128-byte segments 4 KB apart) and re-derive every per-channel constant for each float4. Here a block owns whole ROWS (4 KB contiguous), thread t owns the float4
// column t of every row of its block:
//   stats: per-thread (sum, sumsq) over the block's rows, xor-shuffle over the cpg/4 lanes of a group, then a fixed-order
//          sum over the block's row lanes in shared memory: one partial per (batch, group, block). No atomics anywhere:
//          the result must be bit-identical from run to run (the DDPM loop amplifies a last-bit difference in eps
//          153-fold, and the CUDA-graph and eager paths are tested for equality);
//   apply: the cpg/4 lanes of a group share out the group's partials (all loads in flight at once), shuffle-reduce them
//          to (mean, rstd), fold mean/rstd/gamma/beta/scale/shift of their 4 channels into y = x * a + b ONCE, then
//          stream their rows: one 16-byte load, 4 FMAs (+ SiLU), one 8-byte bf16 (and/or 16-byte fp32) store per row.
//          (A "last block folds the partials" variant of the stats kernel was measured slower: its serial tail sat on
//          the critical path of every GroupNorm.)
// scratch layout (floats): 16 unused | [B][groups][TTB_GN_SPLITS][2] partial sums.
__global__ void __launch_bounds__(256)
gn_stats_rows_kernel(const float* __restrict__ x, int B, int S, int C, int groups, int cpg, int tpr, int rows_per,
                     int splits, float* __restrict__ scratch) {
  pdl_wait();       // (no early PDL trigger: the dependents are scheduled when this grid drains)
  __shared__ float sacc[2 * 256];                               // [row lane][group][2]; rows_par * groups = 256 / lpg
  const int sp = blockIdx.x, b = blockIdx.y;
  const int rows_par = 256 / tpr;
  const int rl = threadIdx.x / tpr, ct = threadIdx.x - rl * tpr;
  const int s0 = sp * rows_per, s1 = min(S, s0 + rows_per);
  const float* xp = x + (long long)b * S * C + ct * 4;
  float s = 0.f, q = 0.f;
  int r = s0 + rl;
  for (; r + 7 * rows_par < s1; r += 8 * rows_par) {           // 8 independent 16-byte loads in flight per thread
    float4 t[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) t[u] = *reinterpret_cast<const float4*>(xp + (long long)(r + u * rows_par) * C);
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      s += (t[u].x + t[u].y) + (t[u].z + t[u].w);
      q += (t[u].x * t[u].x + t[u].y * t[u].y) + (t[u].z * t[u].z + t[u].w * t[u].w);
    }
  }
  for (; r < s1; r += rows_par) {
    const float4 t = *reinterpret_cast<const float4*>(xp + (long long)r * C);
    s += (t.x + t.y) + (t.z + t.w);
    q += (t.x * t.x + t.y * t.y) + (t.z * t.z + t.w * t.w);
  }
  const int lpg = cpg >> 2;                                     // lanes per group: power of two <= min(32, tpr)
  for (int off = lpg >> 1; off > 0; off >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, off);
    q += __shfl_xor_sync(0xffffffffu, q, off);
  }
  if ((ct & (lpg - 1)) == 0) {                                  // exactly one writer per (row lane, group)
    const int g = (ct * 4) / cpg;
    sacc[(rl * groups + g) * 2] = s;
    sacc[(rl * groups + g) * 2 + 1] = q;
  }
  __syncthreads();
  for (int g = threadIdx.x; g < groups; g += 256) {
    float su = 0.f, sq = 0.f;
    for (int k = 0; k < rows_par; ++k) { su += sacc[(k * groups + g) * 2]; sq += sacc[(k * groups + g) * 2 + 1]; }
    float* p = scratch + 16 + (((long long)b * groups + g) * TTB_GN_SPLITS + sp) * 2;
    p[0] = su;
    p[1] = sq;
  }
  (void)B; (void)splits;
}

__global__ void __launch_bounds__(256)
gn_apply_rows_kernel(const float* __restrict__ x, int S, int C, int groups, int cpg, int tpr, int rows_per, int splits,
                     const float* __restrict__ scratch, const float* __restrict__ gamma, const float* __restrict__ beta,
                     const float* __restrict__ ss, int ss_bstride, const int* __restrict__ ss_row, int ss_row_stride,
                     int do_silu, __nv_bfloat16* __restrict__ ob, int ldo, float* __restrict__ of, int ldof, int early) {
  if (early) pdl_launch_dependents();   // TTB_GN_EARLY (default on): as layernorm_warp_kernel, for the GEMM that follows
  pdl_wait();
  const int b = blockIdx.y;
  const int rows_par = 256 / tpr;
  const int rl = threadIdx.x / tpr, ct = threadIdx.x - rl * tpr;
  const int c = ct * 4;
  const int g = c / cpg;
  // (mean, rstd) of this thread's group: the group's lanes take every lpg-th partial each, then a fixed xor tree
  const int lpg = cpg >> 2, sub = ct & (lpg - 1);
  const float2* part = reinterpret_cast<const float2*>(scratch + 16) + ((long long)b * groups + g) * TTB_GN_SPLITS;
  float su = 0.f, sq = 0.f;
  for (int k = sub; k < splits; k += lpg) {
    const float2 p = part[k];
    su += p.x;
    sq += p.y;
  }
  for (int off = lpg >> 1; off > 0; off >>= 1) {
    su += __shfl_xor_sync(0xffffffffu, su, off);
    sq += __shfl_xor_sync(0xffffffffu, sq, off);
  }
  const float n = (float)S * (float)cpg;
  const float mean = su / n;
  const float rstd = rsqrtf(fmaxf(sq / n - mean * mean, 0.f) + 1e-5f);
  float a[4], o[4];
  if (ss && ss_row) ss += (long long)(*ss_row) * ss_row_stride;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    a[j] = rstd * __ldg(gamma + c + j);
    o[j] = __ldg(beta + c + j) - mean * a[j];
    if (ss) {
      const float sc = 1.0f + ss[(long long)b * ss_bstride + c + j], sh = ss[(long long)b * ss_bstride + C + c + j];
      a[j] *= sc;
      o[j] = o[j] * sc + sh;
    }
  }
  const int s0 = blockIdx.x * rows_per, s1 = min(S, s0 + rows_per);
  const float* xp = x + (long long)b * S * C + c;
  for (int r0 = s0 + rl; r0 < s1; r0 += 8 * rows_par) {
    float4 t[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int r = r0 + u * rows_par;
      if (r < s1) t[u] = *reinterpret_cast<const float4*>(xp + (long long)r * C);
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int r = r0 + u * rows_par;
      if (r >= s1) break;
      float y0 = fmaf(t[u].x, a[0], o[0]), y1 = fmaf(t[u].y, a[1], o[1]), y2 = fmaf(t[u].z, a[2], o[2]),
            y3 = fmaf(t[u].w, a[3], o[3]);
      if (do_silu) { y0 = silu(y0); y1 = silu(y1); y2 = silu(y2); y3 = silu(y3); }
      if (ob) *reinterpret_cast<uint2*>(ob + ((long long)b * S + r) * ldo + c) = make_uint2(pack_bf16(y0, y1), pack_bf16(y2, y3));
      if (of) *reinterpret_cast<float4*>(of + ((long long)b * S + r) * ldof + c) = make_float4(y0, y1, y2, y3);
    }
  }
}

}  // namespace ttb
using namespace ttb;

// warp-per-row LayerNorm when the row is NV x 128 floats and everything is 16-byte aligned; false = not applicable
static int gn_early() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("TTB_GN_EARLY"); v = (e && e[0] == '0') ? 0 : 1; }     // default on
  return v;
}

static bool launch_ln_warp(const float* x, int M, int D, const float* g1, const float* b1, const float* g2, const float* b2,
                           __nv_bfloat16* ob, float* of, float* xw, const float* partials, int nsplit,
                           long long split_stride, const float* rbias, cudaStream_t st) {
  const char* impl = getenv("TTB_LN_IMPL");          // "block" forces the block-per-row kernel (A/B timing)
  if (impl && impl[0] == 'b') return false;
  if (D % 128 != 0 || D > 1024 || (split_stride & 3)) return false;
  const void* ptrs[] = {x, g1, b1, g2, b2, ob, of, xw, partials, rbias};
  for (const void* p : ptrs)
    if (p && (reinterpret_cast<uintptr_t>(p) & 15)) return false;
  const dim3 grid((M + 1) / 2);
  static int early = -1;
  if (early < 0) { const char* e = getenv("TTB_LN_EARLY"); early = (e && e[0] == '0') ? 0 : 1; }
#define TTB_LN_CASE(NV)                                                                                              \
  case NV: launch_pdl(layernorm_warp_kernel<NV>, grid, dim3(64), (size_t)0, st, x, M, D, g1, b1, g2, b2, ob, of, xw,  \
                      partials, nsplit, split_stride, rbias, early); break;
  switch (D / 128) {
    TTB_LN_CASE(1) TTB_LN_CASE(2) TTB_LN_CASE(3) TTB_LN_CASE(4) TTB_LN_CASE(5) TTB_LN_CASE(6) TTB_LN_CASE(7) TTB_LN_CASE(8)
    default: return false;
  }
#undef TTB_LN_CASE
  return true;
}

extern "C" int ttb_layernorm(const float* x, int M, int D, const float* g1, const float* b1, const float* g2,
                             const float* b2, void* out_bf16, float* out_f32, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (M <= 0) return 0;
  auto ob = reinterpret_cast<__nv_bfloat16*>(out_bf16);
  if (launch_ln_warp(x, M, D, g1, b1, g2, b2, ob, out_f32, nullptr, nullptr, 0, 0, nullptr, st)) {}
  else if (D <= 1024) layernorm_kernel<4><<<M, 256, 0, st>>>(x, D, g1, b1, g2, b2, ob, out_f32, nullptr, nullptr, 0, 0, nullptr);
  else if (D <= 4096) layernorm_kernel<16><<<M, 256, 0, st>>>(x, D, g1, b1, g2, b2, ob, out_f32, nullptr, nullptr, 0, 0, nullptr);
  else { set_error("ttb_layernorm: D=%d > 4096", D); return -1; }
  TTB_CHECK_LAUNCH("layernorm_kernel");
  return 0;
}

extern "C" int ttb_residual_layernorm(float* x, int M, int D, const float* partials, int nsplit, long long split_stride,
                                      const float* bias, const float* g1, const float* b1, const float* g2,
                                      const float* b2, void* out_bf16, float* out_f32, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (M <= 0) return 0;
  auto ob = reinterpret_cast<__nv_bfloat16*>(out_bf16);
  if (launch_ln_warp(x, M, D, g1, b1, g2, b2, ob, out_f32, x, partials, nsplit, split_stride, bias, st)) {}
  else if (D <= 1024) layernorm_kernel<4><<<M, 256, 0, st>>>(x, D, g1, b1, g2, b2, ob, out_f32, x, partials, nsplit, split_stride, bias);
  else if (D <= 4096) layernorm_kernel<16><<<M, 256, 0, st>>>(x, D, g1, b1, g2, b2, ob, out_f32, x, partials, nsplit, split_stride, bias);
  else { set_error("ttb_residual_layernorm: D=%d > 4096", D); return -1; }
  TTB_CHECK_LAUNCH("layernorm_kernel(residual)");
  return 0;
}

extern "C" int ttb_rmsnorm(const float* x, int M, int D, const float* g, void* out_bf16, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (M <= 0) return 0;
  if (D > 1024) { set_error("ttb_rmsnorm: D=%d > 1024", D); return -1; }
  rmsnorm_kernel<4><<<M, 256, 0, st>>>(x, D, g, reinterpret_cast<__nv_bfloat16*>(out_bf16));
  TTB_CHECK_LAUNCH("rmsnorm_kernel");
  return 0;
}

extern "C" int ttb_groupnorm_apply(const float* x, int B, int S, int C, int groups, const float* gamma, const float* beta,
                                   const float* scale_shift, int ss_bstride, const int* ss_row, int ss_row_stride,
                                   int do_silu, const float* partials, void* out_bf16, int ldo, float* out_f32, int ldof,
                                   void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int splits = (S + 31) / 32;                 // one partial per 32-row block, written by the GEMM epilogue
  if (C != 32 * groups || C > 1024 || (C & (C - 1)) || splits > TTB_GN_SPLITS || S <= 0) {
    set_error("ttb_groupnorm_apply: needs 32 channels per group, C a power of two <= 1024, S <= %d (C=%d groups=%d S=%d)",
              32 * TTB_GN_SPLITS, C, groups, S);
    return -1;
  }
  const int tpr = C >> 2, rows_par = 256 / tpr, rows_per_a = 16 * rows_par;
  launch_pdl(gn_apply_rows_kernel, dim3((S + rows_per_a - 1) / rows_per_a, B), dim3(256), (size_t)0, st,
      x, S, C, groups, 32, tpr, rows_per_a, splits, partials, gamma, beta, scale_shift, ss_bstride, ss_row, ss_row_stride,
      do_silu, reinterpret_cast<__nv_bfloat16*>(out_bf16), ldo, out_f32, ldof, gn_early());
  TTB_CHECK_LAUNCH("gn_apply_rows_kernel");
  return 0;
}

extern "C" int ttb_groupnorm(const float* x, int B, int S, int C, int groups, const float* gamma, const float* beta,
                             const float* scale_shift, int ss_bstride, const int* ss_row, int ss_row_stride,
                             int do_silu, float* partials, void* out_bf16, int ldo, float* out_f32, int ldof,
                             void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (C % groups != 0 || (C & 3)) { set_error("ttb_groupnorm: C=%d groups=%d unsupported", C, groups); return -1; }
  const int cpg = C / groups;
  if (cpg % 4 != 0 && (cpg & 3)) { set_error("ttb_groupnorm: channels per group must be a multiple of 4"); return -1; }
  auto is_pow2 = [](int v) { return v > 0 && (v & (v - 1)) == 0; };
  const int cols = C >> 2, lpg = cpg >> 2;
  const char* impl = getenv("TTB_GN_IMPL");       // "group" forces the generic group-wise kernels (A/B timing)
  const bool force_group = impl && impl[0] == 'g';
  if (!force_group && (cpg & 3) == 0 && is_pow2(cols) && cols <= 256 && is_pow2(lpg) && lpg <= 32 && groups <= 256 && S > 0) {
    // row-wise path (see gn_stats_rows_kernel)
    const int tpr = cols, rows_par = 256 / tpr;
    int splits = (S + 8 * rows_par - 1) / (8 * rows_par);
    splits = splits < 1 ? 1 : (splits > TTB_GN_SPLITS ? TTB_GN_SPLITS : splits);
    const int rows_per_s = (S + splits - 1) / splits;
    splits = (S + rows_per_s - 1) / rows_per_s;
    launch_pdl(gn_stats_rows_kernel, dim3(splits, B), dim3(256), (size_t)0, st, x, B, S, C, groups, cpg, tpr, rows_per_s, splits, partials);
    TTB_CHECK_LAUNCH("gn_stats_rows_kernel");
    const int rows_per_a = 16 * rows_par;     // two batches of 8 loads per thread; amortises the per-block stats fold
    launch_pdl(gn_apply_rows_kernel, dim3((S + rows_per_a - 1) / rows_per_a, B), dim3(256), (size_t)0, st,
        x, S, C, groups, cpg, tpr, rows_per_a, splits, (const float*)partials, gamma, beta, scale_shift, ss_bstride, ss_row, ss_row_stride,
        do_silu, reinterpret_cast<__nv_bfloat16*>(out_bf16), ldo, out_f32, ldof, gn_early());
    TTB_CHECK_LAUNCH("gn_apply_rows_kernel");
    return 0;
  }
  const int splits = 8;      // generic (group-wise) path: any C % 4 == 0
  dim3 g1(groups, splits, B);
  partials += 16;            // keep clear of the row-wise path's ticket at the head of the scratch buffer
  gn_stats_kernel<<<g1, 256, 0, st>>>(x, S, C, cpg, splits, partials);
  TTB_CHECK_LAUNCH("gn_stats_kernel");
  const long long total = (long long)S * (C >> 2);
  dim3 g2((unsigned)((total + 255) / 256), B);
  gn_apply_kernel<<<g2, 256, 0, st>>>(x, S, C, groups, cpg, splits, partials, gamma, beta, scale_shift, ss_bstride,
                                      ss_row, ss_row_stride, do_silu, reinterpret_cast<__nv_bfloat16*>(out_bf16), ldo, out_f32, ldof);
  TTB_CHECK_LAUNCH("gn_apply_kernel");
  return 0;
}
