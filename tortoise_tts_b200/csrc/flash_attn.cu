// wgmma flash attention, head_dim 64, bf16 in/out, fp32 softmax statistics.
//
//   out = softmax(q k^T * scale + relpos_bias[h][kj - qi] (+ causal mask)) v      per (sequence, head)
//
// One CTA = 128 queries of one (sequence, head); KV streamed in tiles of 64 keys by TMA (2 stages) straight out of
// the token-major qkv buffer (3-D tensor map, out-of-range rows zero-filled).
//   warps 0..3, 4..7 : two consumer warpgroups of 64 queries each, sharing every K/V tile. Per tile:
//                      S = Q K^T (wgmma m64n64k16, both operands K-major in shared memory) -> scale/bias/mask and the
//                      running max/sum in registers (a query row lives in the 4 lanes of a quad) -> P (bf16) packed
//                      into the A fragments of O += P V (wgmma with A from registers, B = V tile used MN-major as
//                      loaded). O stays in registers.
//   warp 8           : TMA producer (Q once, then K/V tiles)
// The two warpgroups run independently, so while one does its softmax the tensor core serves the other.
// Replaces the materialised [H, T, T] score tensors of QKVAttentionLegacy (arch_util.py:60-77), HF GPT2Attention._attn
// and xtransformers Attention (xtransformers.py:660-712).
#include <type_traits>

#include "common.cuh"
#include "ttb_internal.h"

namespace ttb {

constexpr int FA_BM = 128;   // queries per CTA
constexpr int FA_BN = 64;    // keys per tile
constexpr int FA_CONSUMERS = 256;
constexpr int FA_PRODUCER_WARP = 8;
constexpr int FA_THREADS = FA_CONSUMERS + 32;
constexpr int FA_STAGES = 2;

struct FaSmem {
  static constexpr int Q_BYTES = FA_BM * 64 * 2;          // 16 KB
  static constexpr int K_BYTES = FA_BN * 64 * 2;          // 8 KB
  static constexpr int V_BYTES = FA_BN * 64 * 2;          // 8 KB
  static constexpr int Q_OFF = 0;
  static constexpr int KV_OFF = Q_BYTES;
  static constexpr int BIAS_OFF = KV_OFF + FA_STAGES * (K_BYTES + V_BYTES);   // 192 floats
  static constexpr int BAR_OFF = BIAS_OFF + 192 * 4;
  static constexpr int TOTAL = BAR_OFF + 16 * 8 + 1024;
};

__global__ void __launch_bounds__(FA_THREADS, 2)
flash_attn_tc_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                     const __grid_constant__ CUtensorMap map_v, TtbAttnArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + FaSmem::BAR_OFF);
  uint64_t* q_full = bars + 0;
  uint64_t* kv_full = bars + 1;            // [FA_STAGES]
  uint64_t* kv_empty = bars + 1 + FA_STAGES;
  float* sbias = reinterpret_cast<float*>(smem + FaSmem::BIAS_OFF);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * FA_BM, h = blockIdx.y, seq = blockIdx.z;
  const int Tq = a.T;                          // queries per sequence
  const int T = a.Tk > 0 ? a.Tk : a.T;         // keys per sequence (bias / causal need Tk == T)
  const int kv_end = a.causal ? min(T, q0 + FA_BM) : T;
  // KV addressing: packed qkv rows (k_off/v_off + 64*h columns, sequence = 3rd coordinate) or a head-major cache
  // [H][Tk][64] shared by every sequence (kv_headmajor): head = 3rd coordinate.
  const int kc0 = a.kv_headmajor ? 0 : a.k_off + h * 64;
  const int vc0 = a.kv_headmajor ? 0 : a.v_off + h * 64;
  const int kvc2 = a.kv_headmajor ? h : seq;
  const int ntiles = (kv_end + FA_BN - 1) / FA_BN;

  if (warp == FA_PRODUCER_WARP && lane == 0) {
    tma_prefetch_desc(&map_q);
    tma_prefetch_desc(&map_k);
    tma_prefetch_desc(&map_v);
    mbar_init(q_full, 1);
    for (int s = 0; s < FA_STAGES; ++s) { mbar_init(&kv_full[s], 1); mbar_init(&kv_empty[s], 2); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();        // barrier init and descriptor prefetch above overlap the tail of the qkv GEMM

  if (warp == FA_PRODUCER_WARP) {
    if (lane == 0) {
      mbar_arrive_expect_tx(q_full, FaSmem::Q_BYTES);
      tma_load_3d(smem + FaSmem::Q_OFF, &map_q, q_full, h * 64, q0, seq);
      int stage = 0; uint32_t phase = 0;
      for (int j = 0; j < ntiles; ++j) {
        mbar_wait(&kv_empty[stage], phase ^ 1);
        uint8_t* sk = smem + FaSmem::KV_OFF + stage * (FaSmem::K_BYTES + FaSmem::V_BYTES);
        uint8_t* sv = sk + FaSmem::K_BYTES;
        mbar_arrive_expect_tx(&kv_full[stage], FaSmem::K_BYTES + FaSmem::V_BYTES);
        tma_load_3d(sk, &map_k, &kv_full[stage], kc0, j * FA_BN, kvc2);
        tma_load_3d(sv, &map_v, &kv_full[stage], vc0, j * FA_BN, kvc2);
        if (++stage == FA_STAGES) { stage = 0; phase ^= 1; }
      }
    }
    __syncwarp();
  } else {
    const int wg = warp >> 2;
    const int g = lane >> 2, t = lane & 3;
    const int row0 = wg * 64 + (warp & 3) * 16 + g;   // this thread's query rows inside the tile: row0 and row0 + 8
    const float sl2 = a.scale * 1.4426950408889634f;
    const float* bias_h = a.bias ? a.bias + (long long)h * (2 * T - 1) + (T - 1) : nullptr;
    // Running statistics in the log2 domain, per row half (hh = 0: row0, 1: row0 + 8); l is this thread's share of the
    // row sum (reduced over the quad at the end). O is rescaled only when a row's max grows by more than 2^8 ("lazy
    // rescale"), so P values stay <= 256.
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    const uint32_t sq = smem_u32(smem + FaSmem::Q_OFF) + wg * (64 * 128);
    mbar_wait(q_full, 0);
    int stage = 0; uint32_t phase = 0;
    for (int j = 0; j < ntiles; ++j) {
      const int k0 = j * FA_BN;
      // Tile classification (uniform over the CTA): far from the diagonal the T5 bias is saturated, i.e. constant
      // over the whole tile, and no key is masked -> one FFMA + one EX2 per score ("fast" tiles).
      const bool nomask = (k0 + FA_BN <= T) && (!a.causal || k0 + FA_BN - 1 <= q0);
      bool cbias_ok = (bias_h == nullptr);
      float cb = 0.f;
      if (bias_h && a.bias_sat > 0) {
        if (k0 - q0 + (FA_BN - 1) <= -a.bias_sat) { cbias_ok = true; cb = __ldg(bias_h - (T - 1)) * 1.4426950408889634f; }
        else if (k0 - q0 - (FA_BM - 1) >= a.bias_sat) { cbias_ok = true; cb = __ldg(bias_h + (T - 1)) * 1.4426950408889634f; }
      }
      const bool fast = nomask && cbias_ok;
      if (bias_h && !fast) {
        // window of the Toeplitz bias table needed by this (q-tile, k-tile): rel = kj - qi in [k0-q0-127, k0-q0+63]
        named_barrier(1, FA_CONSUMERS);                   // previous tile's readers are done
        for (int i = threadIdx.x; i < 191; i += FA_CONSUMERS) {
          const int rel = k0 - q0 - 127 + i;
          sbias[i] = (rel > -T && rel < T) ? __ldg(bias_h + rel) * 1.4426950408889634f : 0.f;
        }
        named_barrier(1, FA_CONSUMERS);
      }
      mbar_wait(&kv_full[stage], phase);
      const uint32_t sk = smem_u32(smem + FaSmem::KV_OFF + stage * (FaSmem::K_BYTES + FaSmem::V_BYTES));
      const uint32_t sv = sk + FaSmem::K_BYTES;
      // S[64 x 64 keys] = Q[64 x 64d] K[64 keys x 64d]^T
      float s[32];
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_m64n64k16_bf16_ss(s, wgmma_desc_kmajor_sw128(sq + k * 32), wgmma_desc_kmajor_sw128(sk + k * 32), k != 0);
      wgmma_commit();
      wgmma_wait<0>();
      // register i: row half (i >> 1) & 1, key column c = 8 (i >> 2) + 2 t + (i & 1)
      float mx[2] = {-INFINITY, -INFINITY};
      if (fast) {
#pragma unroll
        for (int i = 0; i < 32; ++i) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], s[i]);
        mx[0] = fmaf(mx[0], sl2, cb);
        mx[1] = fmaf(mx[1], sl2, cb);
      } else {
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const int hh = (i >> 1) & 1;
          const int row = row0 + 8 * hh;
          const int c = 8 * (i >> 2) + 2 * t + (i & 1);
          const int klim = min(T - k0, a.causal ? (q0 + row - k0 + 1) : FA_BN);   // keys c < klim are visible to this row
          float v = s[i] * sl2;
          if (bias_h) v += sbias[c - row + 127];
          v = (c < klim) ? v : -INFINITY;
          s[i] = v;
          mx[hh] = fmaxf(mx[hh], v);
        }
      }
      float corr[2], cm[2];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
        mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
        const bool grow = mx[hh] > m[hh] + 8.0f;         // also true for the first finite max (m = -inf)
        const float m_new = grow ? mx[hh] : m[hh];
        corr[hh] = grow ? exp2f(m[hh] - m_new) : 1.0f;   // exp2(-inf) = 0 on the first tile
        m[hh] = m_new;
        const float m_use = (m_new == -INFINITY) ? 0.f : m_new;
        cm[hh] = fast ? cb - m_use : -m_use;
      }
      float psum[2] = {0.f, 0.f};
      uint32_t pa[16];                                    // P as the A fragments of the four k16 steps of P V
#pragma unroll
      for (int i = 0; i < 32; i += 2) {
        const int hh = (i >> 1) & 1;
        const float p0 = fast ? exp2f(fmaf(s[i], sl2, cm[hh])) : exp2f(s[i] + cm[hh]);
        const float p1 = fast ? exp2f(fmaf(s[i + 1], sl2, cm[hh])) : exp2f(s[i + 1] + cm[hh]);
        psum[hh] += p0 + p1;
        pa[i >> 1] = pack_bf16(p0, p1);
      }
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) l[hh] = l[hh] * corr[hh] + psum[hh];
#pragma unroll
      for (int i = 0; i < 32; ++i) o[i] *= corr[(i >> 1) & 1];
      // O[64 x 64d] += P[64 x 64 keys] V[64 keys x 64d]; the key index advances 16 rows of 128 B per step in the V tile
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_m64n64k16_bf16_rs<1>(o, pa + 4 * k, wgmma_desc_mnmajor_sw128(sv + k * 2048, 0), 1u);
      wgmma_commit();
      wgmma_wait<0>();
      if ((threadIdx.x & 127) == 0) mbar_arrive(&kv_empty[stage]);
      if (++stage == FA_STAGES) { stage = 0; phase ^= 1; }
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
      l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
      const int qi = q0 + row0 + 8 * hh;
      if (qi >= Tq) continue;
      const float inv = 1.0f / l[hh];
      if (a.lse) {
        // partial-attention mode: normalised O in fp32 + log2-sum-exp, to be merged with another key range
        float* op = a.out_f32 + ((long long)seq * Tq + qi) * a.ldo + h * 64 + 2 * t;
#pragma unroll
        for (int nb = 0; nb < 8; ++nb)
          *reinterpret_cast<float2*>(op + 8 * nb) = make_float2(o[4 * nb + 2 * hh] * inv, o[4 * nb + 2 * hh + 1] * inv);
        if (t == 0) a.lse[((long long)seq * Tq + qi) * a.H + h] = m[hh] + log2f(l[hh]);
      } else {
        __nv_bfloat16* op = reinterpret_cast<__nv_bfloat16*>(a.out) + ((long long)seq * Tq + qi) * a.ldo + h * 64 + 2 * t;
#pragma unroll
        for (int nb = 0; nb < 8; ++nb)
          *reinterpret_cast<uint32_t*>(op + 8 * nb) = pack_bf16(o[4 * nb + 2 * hh] * inv, o[4 * nb + 2 * hh + 1] * inv);
      }
    }
  }
  pdl_launch_dependents();
}

bool flash_attention_supported(const TtbAttnArgs& a) {
  if (a.kv || a.lse) return true;      // split Q / KV tensors and LSE output exist only in the wgmma kernel
  return a.T >= 64 && (a.ld % 8) == 0;
}

int flash_attention_launch(const TtbAttnArgs& a, cudaStream_t st) {
  CUtensorMap mq, mk, mv;
  if (get_tensor_map_bf16(&mq, a.qkv, (uint64_t)a.ld, (uint64_t)a.T, (uint64_t)a.nseq, (uint64_t)a.ld,
                          (uint64_t)a.T * a.ld, 64, FA_BM)) return -1;
  if (a.kv_headmajor) {
    if (!a.kv || !a.kv_v || a.Tk <= 0 || a.causal || a.bias) { set_error("flash attention: bad head-major KV arguments"); return -1; }
    if (get_tensor_map_bf16(&mk, a.kv, 64, (uint64_t)a.Tk, (uint64_t)a.H, 64, (uint64_t)a.Tk * 64, 64, FA_BN)) return -1;
    if (get_tensor_map_bf16(&mv, a.kv_v, 64, (uint64_t)a.Tk, (uint64_t)a.H, 64, (uint64_t)a.Tk * 64, 64, FA_BN)) return -1;
  } else {
    if (a.Tk > 0 && a.Tk != a.T) { set_error("flash attention: Tk != T needs the head-major KV form"); return -1; }
    if (get_tensor_map_bf16(&mk, a.qkv, (uint64_t)a.ld, (uint64_t)a.T, (uint64_t)a.nseq, (uint64_t)a.ld,
                            (uint64_t)a.T * a.ld, 64, FA_BN)) return -1;
    mv = mk;
  }
  if (a.lse && !a.out_f32) { set_error("flash attention: lse output needs out_f32"); return -1; }
  static bool attr = false;
  if (!attr) {
    cudaError_t r = cudaFuncSetAttribute(flash_attn_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FaSmem::TOTAL);
    if (r != cudaSuccess) return check_cuda(r, "cudaFuncSetAttribute(flash_attn)");
    attr = true;
  }
  dim3 grid((a.T + FA_BM - 1) / FA_BM, a.H, a.nseq);
  const cudaError_t le = launch_pdl(flash_attn_tc_kernel, grid, dim3(FA_THREADS), (size_t)FaSmem::TOTAL, st, mq, mk, mv, a);
  if (le != cudaSuccess) return check_cuda(le, "flash_attn_tc_kernel launch");
  TTB_CHECK_LAUNCH("flash_attn_tc_kernel");
  return 0;
}

}  // namespace ttb
