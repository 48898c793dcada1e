// Attention kernels, head_dim 64.
//  * attn_simt_kernel: general softmax(q k^T * scale + relpos_bias [+ causal]) v, online-softmax (flash) form,
//    one query per thread, K/V tiles staged in shared memory as fp32. Used for prompt prefill, latents, CLVP and
//    diffusion attention (the wgmma path in flash_attn.cu takes the large shapes).
//  * ar_decode_attn_kernel: single-query attention of every (candidate, head) over [shared prefix | own KV]
//    for the GPT-2 sampler; memory-bound on the KV stream (HBM roofline), appends the new K/V.
#include "common.cuh"
#include "ttb_internal.h"
#include <cstring>

namespace ttb {

constexpr int ATT_Q = 128;   // queries per block (one per thread)
constexpr int ATT_KT = 32;   // keys per tile

__global__ void __launch_bounds__(ATT_Q)
attn_simt_kernel(TtbAttnArgs a) {
  __shared__ __align__(16) float sk[ATT_KT][64];
  __shared__ __align__(16) float sv[ATT_KT][64];
  const int h = blockIdx.y, seq = blockIdx.z;
  const int q0 = blockIdx.x * ATT_Q;
  const int qi = q0 + threadIdx.x;
  const bool active = qi < a.T;
  const __nv_bfloat16* base = reinterpret_cast<const __nv_bfloat16*>(a.qkv) + (long long)seq * a.T * a.ld + h * 64;
  float q[64], o[64];
#pragma unroll
  for (int d = 0; d < 64; ++d) o[d] = 0.f;
  if (active) {
    const uint4* qp = reinterpret_cast<const uint4*>(base + (long long)qi * a.ld);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      uint4 u = qp[i];
      float2 f0 = unpack_bf16(u.x), f1 = unpack_bf16(u.y), f2 = unpack_bf16(u.z), f3 = unpack_bf16(u.w);
      q[8 * i] = f0.x * a.scale; q[8 * i + 1] = f0.y * a.scale; q[8 * i + 2] = f1.x * a.scale; q[8 * i + 3] = f1.y * a.scale;
      q[8 * i + 4] = f2.x * a.scale; q[8 * i + 5] = f2.y * a.scale; q[8 * i + 6] = f3.x * a.scale; q[8 * i + 7] = f3.y * a.scale;
    }
  } else {
#pragma unroll
    for (int d = 0; d < 64; ++d) q[d] = 0.f;
  }
  float mrun = -INFINITY, lrun = 0.f;
  const int kend = a.causal ? min(a.T, q0 + ATT_Q) : a.T;
  const float* bias = a.bias ? a.bias + (long long)h * (2 * a.T - 1) + (a.T - 1) : nullptr;
  for (int k0 = 0; k0 < kend; k0 += ATT_KT) {
    __syncthreads();
    // cooperative load of K and V tiles: ATT_KT rows x 64 dims, 8 bf16 per uint4 -> 8 uint4 per row
    for (int i = threadIdx.x; i < ATT_KT * 8; i += ATT_Q) {
      const int r = i >> 3, c = (i & 7) * 8;
      const int kj = k0 + r;
      uint4 uk = make_uint4(0, 0, 0, 0), uv = make_uint4(0, 0, 0, 0);
      if (kj < a.T) {
        uk = *reinterpret_cast<const uint4*>(base + (long long)kj * a.ld + a.k_off + c);
        uv = *reinterpret_cast<const uint4*>(base + (long long)kj * a.ld + a.v_off + c);
      }
      float2 t;
      t = unpack_bf16(uk.x); sk[r][c] = t.x; sk[r][c + 1] = t.y;
      t = unpack_bf16(uk.y); sk[r][c + 2] = t.x; sk[r][c + 3] = t.y;
      t = unpack_bf16(uk.z); sk[r][c + 4] = t.x; sk[r][c + 5] = t.y;
      t = unpack_bf16(uk.w); sk[r][c + 6] = t.x; sk[r][c + 7] = t.y;
      t = unpack_bf16(uv.x); sv[r][c] = t.x; sv[r][c + 1] = t.y;
      t = unpack_bf16(uv.y); sv[r][c + 2] = t.x; sv[r][c + 3] = t.y;
      t = unpack_bf16(uv.z); sv[r][c + 4] = t.x; sv[r][c + 5] = t.y;
      t = unpack_bf16(uv.w); sv[r][c + 6] = t.x; sv[r][c + 7] = t.y;
    }
    __syncthreads();
    if (!active) continue;
    float s[ATT_KT];
    float tmax = -INFINITY;
#pragma unroll
    for (int j = 0; j < ATT_KT; ++j) {
      const float4* kr = reinterpret_cast<const float4*>(&sk[j][0]);
      float acc = 0.f;
#pragma unroll
      for (int d = 0; d < 16; ++d) {
        float4 kk = kr[d];
        acc += q[4 * d] * kk.x + q[4 * d + 1] * kk.y + q[4 * d + 2] * kk.z + q[4 * d + 3] * kk.w;
      }
      const int kj = k0 + j;
      if (bias && kj < a.T) acc += __ldg(bias + (kj - qi));
      const bool ok = (kj < a.T) && (!a.causal || kj <= qi);
      s[j] = ok ? acc : -INFINITY;
      tmax = fmaxf(tmax, s[j]);
    }
    const float mnew = fmaxf(mrun, tmax);
    if (mnew == -INFINITY) continue;
    const float corr = __expf(mrun - mnew);
    lrun *= corr;
#pragma unroll
    for (int d = 0; d < 64; ++d) o[d] *= corr;
#pragma unroll
    for (int j = 0; j < ATT_KT; ++j) {
      const float p = __expf(s[j] - mnew);
      lrun += p;
      const float4* vr = reinterpret_cast<const float4*>(&sv[j][0]);
#pragma unroll
      for (int d = 0; d < 16; ++d) {
        float4 vv = vr[d];
        o[4 * d] += p * vv.x; o[4 * d + 1] += p * vv.y; o[4 * d + 2] += p * vv.z; o[4 * d + 3] += p * vv.w;
      }
    }
    mrun = mnew;
  }
  if (active) {
    const float inv = 1.0f / lrun;
    __nv_bfloat16* op = reinterpret_cast<__nv_bfloat16*>(a.out) + ((long long)seq * a.T + qi) * a.ldo + h * 64;
    uint4* o4 = reinterpret_cast<uint4*>(op);
#pragma unroll
    for (int i = 0; i < 8; ++i)
      o4[i] = make_uint4(pack_bf16(o[8 * i] * inv, o[8 * i + 1] * inv), pack_bf16(o[8 * i + 2] * inv, o[8 * i + 3] * inv),
                         pack_bf16(o[8 * i + 4] * inv, o[8 * i + 5] * inv), pack_bf16(o[8 * i + 6] * inv, o[8 * i + 7] * inv));
  }
}

// ------------------------------------------------------------------ small general attention (any head_dim = 32 * DPL)
// One warp per query; lane l holds dims [l*DPL, (l+1)*DPL) of q and of the output row. Used where head_dim != 64 and the
// sequences are short: the diffusion contextual embedder (C = 2048, 16 heads of 128, T = 101 per clip;
// models/diffusion_decoder.py:186-192 with QKVAttentionLegacy, arch_util.py:44-77).
template <int DPL>
__global__ void __launch_bounds__(128)
attn_warp_kernel(TtbAttnArgs a) {
  const int HD = 32 * DPL;
  const int lane = threadIdx.x & 31;
  const int qi = blockIdx.x * 4 + (threadIdx.x >> 5);
  const int h = blockIdx.y, seq = blockIdx.z;
  if (qi >= a.T) return;
  const __nv_bfloat16* base = reinterpret_cast<const __nv_bfloat16*>(a.qkv) + (long long)seq * a.T * a.ld + h * HD + lane * DPL;
  float q[DPL], o[DPL];
#pragma unroll
  for (int d = 0; d < DPL; ++d) { q[d] = __bfloat162float(base[(long long)qi * a.ld + d]) * a.scale; o[d] = 0.f; }
  const float* bias = a.bias ? a.bias + (long long)h * (2 * a.T - 1) + (a.T - 1) : nullptr;
  float m = -INFINITY, l = 0.f;
  const int kend = a.causal ? qi + 1 : a.T;
  for (int kj = 0; kj < kend; ++kj) {
    const __nv_bfloat16* kr = base + (long long)kj * a.ld + a.k_off;
    const __nv_bfloat16* vr = base + (long long)kj * a.ld + a.v_off;
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < DPL; ++d) s = fmaf(q[d], __bfloat162float(kr[d]), s);
    s = warp_sum(s);
    if (bias) s += __ldg(bias + (kj - qi));
    const float m_new = fmaxf(m, s);
    const float corr = __expf(m - m_new);
    const float p = __expf(s - m_new);
    l = l * corr + p;
#pragma unroll
    for (int d = 0; d < DPL; ++d) o[d] = o[d] * corr + p * __bfloat162float(vr[d]);
    m = m_new;
  }
  const float inv = 1.0f / l;
  __nv_bfloat16* op = reinterpret_cast<__nv_bfloat16*>(a.out) + ((long long)seq * a.T + qi) * a.ldo + h * HD + lane * DPL;
#pragma unroll
  for (int d = 0; d < DPL; ++d) op[d] = __float2bfloat16(o[d] * inv);
}

// ------------------------------------------------------------------ AR decode attention
// Single-query attention of every (candidate, head) over [shared prompt prefix | the candidate's own KV] with online
// softmax (flash-decoding form). grid (H, ceil(B/8)); 8 warps per block, ONE CANDIDATE PER WARP, all on the same head:
//   * the prefix K/V of this head is staged tile by tile (64 positions, 16 KB) in shared memory ONCE per block and
//     reused by the 8 candidates (the prefix is identical for all candidates: 8x less L2->SM traffic);
//   * the candidate's own KV is streamed from HBM with 16-byte loads: a warp instruction covers 4 positions x 8
//     dim-chunks (512 contiguous bytes), 4 K + 4 V instructions in flight per iteration;
//   * lane = (psub = position within the group of 4, dch = 8-dim chunk); the q.k dot product is reduced over the 8
//     dch lanes with shuffles; every psub group keeps its own running (max, sum, acc[8]) which are merged at the end.
// The new token's K/V is appended to the cache by the owning warp first.
constexpr int DEC_WARPS = 8;
constexpr int DEC_THREADS = DEC_WARPS * 32;
constexpr int DEC_PT = 64;   // prefix positions per shared-memory tile

struct DecState { float m, l; float acc[8]; };

TTB_DEVINL void dec_update(DecState& st, float s, bool ok, const uint4& vv) {
  // s is already in the log2 domain
  const float sm = ok ? s : -INFINITY;
  const float m_new = fmaxf(st.m, sm);
  const float m_use = (m_new == -INFINITY) ? 0.f : m_new;
  const float corr = exp2f(st.m - m_use);
  const float p = exp2f(sm - m_use);
  st.l = st.l * corr + p;
  st.m = m_new;
  const float2 f0 = unpack_bf16(vv.x), f1 = unpack_bf16(vv.y), f2 = unpack_bf16(vv.z), f3 = unpack_bf16(vv.w);
  st.acc[0] = st.acc[0] * corr + p * f0.x; st.acc[1] = st.acc[1] * corr + p * f0.y;
  st.acc[2] = st.acc[2] * corr + p * f1.x; st.acc[3] = st.acc[3] * corr + p * f1.y;
  st.acc[4] = st.acc[4] * corr + p * f2.x; st.acc[5] = st.acc[5] * corr + p * f2.y;
  st.acc[6] = st.acc[6] * corr + p * f3.x; st.acc[7] = st.acc[7] * corr + p * f3.y;
}

TTB_DEVINL float dec_dot(const float* q, const uint4& kk) {
  const float2 f0 = unpack_bf16(kk.x), f1 = unpack_bf16(kk.y), f2 = unpack_bf16(kk.z), f3 = unpack_bf16(kk.w);
  float d = q[0] * f0.x + q[1] * f0.y + q[2] * f1.x + q[3] * f1.y + q[4] * f2.x + q[5] * f2.y + q[6] * f3.x + q[7] * f3.y;
  d += __shfl_xor_sync(0xffffffffu, d, 1);
  d += __shfl_xor_sync(0xffffffffu, d, 2);
  d += __shfl_xor_sync(0xffffffffu, d, 4);
  return d;
}

__global__ void __launch_bounds__(DEC_THREADS, 4)
ar_decode_attn_kernel(const __nv_bfloat16* __restrict__ qkv, const __nv_bfloat16* __restrict__ pk,
                      const __nv_bfloat16* __restrict__ pv, __nv_bfloat16* __restrict__ ck,
                      __nv_bfloat16* __restrict__ cv, const TtbArState* __restrict__ state, int B, int H, int P, int Nmax,
                      float* __restrict__ o_c, float* __restrict__ lse_c) {
  pdl_wait();
  const int h = blockIdx.x;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.y * DEC_WARPS + w;
  const bool active = b < B;
  const int psub = lane >> 3, dch = lane & 7;
  const int D = H * 64;
  // decode step t (>= 1) feeds token t-1 whose K/V land in candidate slot t-1
  const int slot = state->step - 1;
  const int nc = slot + 1;                     // candidate entries incl. the new one
  __nv_bfloat16* ckb = ck + ((long long)(active ? b : 0) * H + h) * Nmax * 64;
  __nv_bfloat16* cvb = cv + ((long long)(active ? b : 0) * H + h) * Nmax * 64;
  float q[8];
  {
    const __nv_bfloat16* row = qkv + (long long)(active ? b : 0) * 3 * D + h * 64;
    const uint4 uq = reinterpret_cast<const uint4*>(row)[dch];
    const float sc = 0.125f * 1.4426950408889634f;     // 1/sqrt(64) and log2(e)
    const float2 f0 = unpack_bf16(uq.x), f1 = unpack_bf16(uq.y), f2 = unpack_bf16(uq.z), f3 = unpack_bf16(uq.w);
    q[0] = f0.x * sc; q[1] = f0.y * sc; q[2] = f1.x * sc; q[3] = f1.y * sc;
    q[4] = f2.x * sc; q[5] = f2.y * sc; q[6] = f3.x * sc; q[7] = f3.y * sc;
    if (active && lane < 16) {                   // append the new K (lanes 0-7) and V (lanes 8-15) rows
      const uint4 nv = reinterpret_cast<const uint4*>(row + (lane < 8 ? D : 2 * D))[dch];
      reinterpret_cast<uint4*>((lane < 8 ? ckb : cvb) + (long long)slot * 64)[dch] = nv;
    }
  }
  // The shared-prompt part of the context is handled concurrently on the tensor cores (flash_attn_tc_kernel over the
  // prefix cache, forked onto a side stream by the host wrapper); this kernel covers the candidate's own keys and
  // emits a partial (normalised row, log2-sum-exp) that ar_attn_merge_kernel combines with the prefix partial.
  DecState st;
  st.m = -INFINITY; st.l = 0.f;
#pragma unroll
  for (int d = 0; d < 8; ++d) st.acc[d] = 0.f;
  // ---- phase B: the candidate's own KV, streamed from global memory
  __syncwarp();
  // Software-pipelined: the loads of batch i+1 (8 positions: 2 K + 2 V 16-byte loads per lane) are issued before the
  // math of batch i, so every warp keeps 4 KB in flight continuously instead of alternating load / compute phases.
  if (active) {
    constexpr int U = 2;
    uint4 kk[U], vv[U], kn[U], vn[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int j = u * 4 + psub;
      const bool ok = j < nc;
      kk[u] = ok ? reinterpret_cast<const uint4*>(ckb + (long long)j * 64)[dch] : make_uint4(0, 0, 0, 0);
      vv[u] = ok ? reinterpret_cast<const uint4*>(cvb + (long long)j * 64)[dch] : make_uint4(0, 0, 0, 0);
    }
    for (int j0 = 0; j0 < nc; j0 += 4 * U) {
      const int jn = j0 + 4 * U;
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int j = jn + u * 4 + psub;
        const bool ok = j < nc;
        kn[u] = ok ? reinterpret_cast<const uint4*>(ckb + (long long)j * 64)[dch] : make_uint4(0, 0, 0, 0);
        vn[u] = ok ? reinterpret_cast<const uint4*>(cvb + (long long)j * 64)[dch] : make_uint4(0, 0, 0, 0);
      }
      // one shared running-max update for the batch (fewer dependent EX2 than per-position updates)
      float s[U];
      float bm = -INFINITY;
#pragma unroll
      for (int u = 0; u < U; ++u) {
        s[u] = dec_dot(q, kk[u]);
        s[u] = (j0 + u * 4 + psub < nc) ? s[u] : -INFINITY;
        bm = fmaxf(bm, s[u]);
      }
      const float m_new = fmaxf(st.m, bm);
      const float m_use = (m_new == -INFINITY) ? 0.f : m_new;
      const float corr = exp2f(st.m - m_use);
      st.m = m_new;
      st.l *= corr;
#pragma unroll
      for (int d = 0; d < 8; ++d) st.acc[d] *= corr;
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const float p = exp2f(s[u] - m_use);
        st.l += p;
        const float2 f0 = unpack_bf16(vv[u].x), f1 = unpack_bf16(vv[u].y), f2 = unpack_bf16(vv[u].z), f3 = unpack_bf16(vv[u].w);
        st.acc[0] += p * f0.x; st.acc[1] += p * f0.y; st.acc[2] += p * f1.x; st.acc[3] += p * f1.y;
        st.acc[4] += p * f2.x; st.acc[5] += p * f2.y; st.acc[6] += p * f3.x; st.acc[7] += p * f3.y;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) { kk[u] = kn[u]; vv[u] = vn[u]; }
    }
  }
  // ---- merge the 4 position sub-streams (lanes differing in bits 3,4), then normalise
#pragma unroll
  for (int off = 8; off <= 16; off <<= 1) {
    const float m_o = __shfl_xor_sync(0xffffffffu, st.m, off);
    const float l_o = __shfl_xor_sync(0xffffffffu, st.l, off);
    const float m_new = fmaxf(st.m, m_o);
    const float m_use = (m_new == -INFINITY) ? 0.f : m_new;
    const float c_s = exp2f(st.m - m_use), c_o = exp2f(m_o - m_use);
    st.l = st.l * c_s + l_o * c_o;
#pragma unroll
    for (int d = 0; d < 8; ++d) {
      const float a_o = __shfl_xor_sync(0xffffffffu, st.acc[d], off);
      st.acc[d] = st.acc[d] * c_s + a_o * c_o;
    }
    st.m = m_new;
  }
  if (active && psub == 0) {
    // partial result over the candidate's own keys: normalised fp32 row + log2-sum-exp (merged with the prefix part)
    const float inv = 1.0f / st.l;
    float4* op = reinterpret_cast<float4*>(o_c + (long long)b * D + h * 64 + dch * 8);
    op[0] = make_float4(st.acc[0] * inv, st.acc[1] * inv, st.acc[2] * inv, st.acc[3] * inv);
    op[1] = make_float4(st.acc[4] * inv, st.acc[5] * inv, st.acc[6] * inv, st.acc[7] * inv);
    if (dch == 0) lse_c[(long long)b * H + h] = st.m + log2f(st.l);
  }
}

// out = softmax-merge of two partial attentions over disjoint key ranges: (o_p, lse_p) and (o_c, lse_c)
__global__ void ar_attn_merge_kernel(const float* __restrict__ o_p, const float* __restrict__ lse_p,
                                     const float* __restrict__ o_c, const float* __restrict__ lse_c, int B, int H,
                                     __nv_bfloat16* __restrict__ out) {
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // over B * H * 16 (4 dims each)
  if (i >= (long long)B * H * 16) return;
  const long long bh = i >> 4;
  const int c = (int)(i & 15) * 4;
  const float lp = lse_p[bh], lc = lse_c[bh];
  const float mx = fmaxf(lp, lc);
  const float wp = exp2f(lp - mx), wc = exp2f(lc - mx);
  const float inv = 1.0f / (wp + wc);
  const float4 a = *reinterpret_cast<const float4*>(o_p + bh * 64 + c);
  const float4 d = *reinterpret_cast<const float4*>(o_c + bh * 64 + c);
  uint2 o = make_uint2(pack_bf16((a.x * wp + d.x * wc) * inv, (a.y * wp + d.y * wc) * inv),
                       pack_bf16((a.z * wp + d.z * wc) * inv, (a.w * wp + d.w * wc) * inv));
  *reinterpret_cast<uint2*>(out + bh * 64 + c) = o;
}

__global__ void ar_store_prefix_kernel(const __nv_bfloat16* __restrict__ qkv, int P, int H, __nv_bfloat16* __restrict__ pk,
                                       __nv_bfloat16* __restrict__ pv) {
  const int D = H * 64;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // over P * D
  if (i >= (long long)P * D) return;
  const int p = (int)(i / D), c = (int)(i - (long long)p * D);
  const int h = c >> 6, d = c & 63;
  pk[((long long)h * P + p) * 64 + d] = qkv[(long long)p * 3 * D + D + c];
  pv[((long long)h * P + p) * 64 + d] = qkv[(long long)p * 3 * D + 2 * D + c];
}

}  // namespace ttb
using namespace ttb;

extern "C" int ttb_attention(const TtbAttnArgs* ap, void* stream) {
  const TtbAttnArgs& a = *ap;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (a.T <= 0 || a.nseq <= 0) return 0;
  if ((a.ld & 7) || (a.ldo & 7) || (a.k_off & 7) || (a.v_off & 7)) { set_error("ttb_attention: strides must be multiples of 8"); return -1; }
  if (a.head_dim != 0 && a.head_dim != 64) {
    if (a.kv || a.lse || a.out_f32) { set_error("ttb_attention: head_dim %d supports the packed form only", a.head_dim); return -1; }
    dim3 grid((a.T + 3) / 4, a.H, a.nseq);
    switch (a.head_dim) {
      case 32: attn_warp_kernel<1><<<grid, 128, 0, st>>>(a); break;
      case 96: attn_warp_kernel<3><<<grid, 128, 0, st>>>(a); break;
      case 128: attn_warp_kernel<4><<<grid, 128, 0, st>>>(a); break;
      default: set_error("ttb_attention: head_dim %d unsupported (32, 64, 96, 128)", a.head_dim); return -1;
    }
    TTB_CHECK_LAUNCH("attn_warp_kernel");
    return 0;
  }
  if (flash_attention_supported(a)) return flash_attention_launch(a, st);
  dim3 grid((a.T + ATT_Q - 1) / ATT_Q, a.H, a.nseq);
  attn_simt_kernel<<<grid, ATT_Q, 0, st>>>(a);
  TTB_CHECK_LAUNCH("attn_simt_kernel");
  return 0;
}

namespace {
struct ForkJoin {
  cudaStream_t side = nullptr;
  cudaEvent_t fork = nullptr, join = nullptr;
  int init() {
    if (side) return 0;
    if (cudaStreamCreateWithFlags(&side, cudaStreamNonBlocking) != cudaSuccess) return -1;
    if (cudaEventCreateWithFlags(&fork, cudaEventDisableTiming) != cudaSuccess) return -1;
    if (cudaEventCreateWithFlags(&join, cudaEventDisableTiming) != cudaSuccess) return -1;
    return 0;
  }
};
ForkJoin g_fj;
}  // namespace

extern "C" int ttb_ar_decode_attention(const void* qkv, const void* prefix_k, const void* prefix_v, void* cand_k,
                                       void* cand_v, const TtbArState* state, int B, int H, int P, int Nmax, void* out,
                                       float* scratch_o, float* scratch_lse, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (g_fj.init()) { set_error("ttb_ar_decode_attention: cannot create the side stream"); return -2; }
  float* o_p = scratch_o;
  float* o_c = scratch_o + (long long)B * H * 64;
  float* lse_p = scratch_lse;
  float* lse_c = scratch_lse + (long long)B * H;
  // fork: (1) shared prompt prefix = dense [B candidates x P keys] attention per head on the tensor cores (side stream;
  // latency-bound, 2x16 CTAs) runs concurrently with (2) the HBM-bound stream over every candidate's own KV.
  cudaError_t e = cudaEventRecord(g_fj.fork, st);
  if (e == cudaSuccess) e = cudaStreamWaitEvent(g_fj.side, g_fj.fork, 0);
  if (e != cudaSuccess) return check_cuda(e, "decode attention fork");
  TtbAttnArgs a;
  memset(&a, 0, sizeof(a));
  a.qkv = qkv; a.nseq = 1; a.T = B; a.H = H; a.ld = 3 * H * 64; a.ldo = H * 64;
  a.scale = 0.125f; a.kv = prefix_k; a.kv_v = prefix_v; a.kv_headmajor = 1; a.Tk = P;
  a.out_f32 = o_p; a.lse = lse_p;
  if (flash_attention_launch(a, g_fj.side)) return -1;
  dim3 grid(H, (B + DEC_WARPS - 1) / DEC_WARPS);
  const cudaError_t le1 = launch_pdl(ar_decode_attn_kernel, grid, dim3(DEC_THREADS), (size_t)0, st,
      reinterpret_cast<const __nv_bfloat16*>(qkv), reinterpret_cast<const __nv_bfloat16*>(prefix_k),
      reinterpret_cast<const __nv_bfloat16*>(prefix_v), reinterpret_cast<__nv_bfloat16*>(cand_k),
      reinterpret_cast<__nv_bfloat16*>(cand_v), state, B, H, P, Nmax, o_c, lse_c);
  if (le1 != cudaSuccess) return check_cuda(le1, "ar_decode_attn_kernel launch");
  TTB_CHECK_LAUNCH("ar_decode_attn_kernel");
  // join, then merge the two partials
  e = cudaEventRecord(g_fj.join, g_fj.side);
  if (e == cudaSuccess) e = cudaStreamWaitEvent(st, g_fj.join, 0);
  if (e != cudaSuccess) return check_cuda(e, "decode attention join");
  const long long n = (long long)B * H * 16;
  const cudaError_t le2 = launch_pdl(ar_attn_merge_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), (size_t)0, st, o_p, lse_p,
                                     o_c, lse_c, B, H, reinterpret_cast<__nv_bfloat16*>(out));
  if (le2 != cudaSuccess) return check_cuda(le2, "ar_attn_merge_kernel launch");
  TTB_CHECK_LAUNCH("ar_attn_merge_kernel");
  return 0;
}

extern "C" int ttb_ar_store_prefix(const void* qkv, int P, int H, void* prefix_k, void* prefix_v, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long n = (long long)P * H * 64;
  ar_store_prefix_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(qkv), P, H,
                                                                     reinterpret_cast<__nv_bfloat16*>(prefix_k),
                                                                     reinterpret_cast<__nv_bfloat16*>(prefix_v));
  TTB_CHECK_LAUNCH("ar_store_prefix_kernel");
  return 0;
}
