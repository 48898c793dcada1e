// One GPT-2 decode step of the UnifiedVoice sampler as ONE persistent kernel (sm_90a).
//
// Replaces, per generated token, GPT2InferenceModel.forward (models/autoregressive.py:108-186) + the 30 HF GPT2Block
// forwards behind it + final_norm + mel_head for ALL candidates of the batch. As a CUDA graph of ~275
// kernels (LN, 4 skinny GEMMs, 3 attention kernels per layer) the launch chain, not bytes or flops, bounds the step.
// Here the whole step is one cooperative launch of one CTA per SM that walks
// the layer phases with grid-wide barriers:
//
//   embed + ln_1 | for each layer: QKV GEMM | attention (+KV append) | c_proj GEMM | residual + ln_2 | c_fc GEMM + gelu_new
//                |                 mlp.c_proj GEMM | residual + next ln_1 (or ln_f -> final_norm) | ... | mel_head GEMM
//
// GEMM phases ("swap-AB" skinny GEMM): the WEIGHT rows are the wgmma M dimension (128-row tiles streamed once from HBM by
// TMA, 64 rows per consumer warpgroup) and the candidate batch is the wgmma N dimension (16..128 columns), so a 32-candidate step does not pay for a
// 128-row activation tile. Work items = (row tile, batch tile, K split); split-K partials are reduced in a fixed order
// by the last CTA to finish a tile (ticket counter), which also applies bias / gelu_new and writes the bf16 result, or
// - for the two GEMMs that feed the residual stream - by the LayerNorm phase that follows.
// Attention phase: K|V of a candidate are interleaved per position ([pos][K 64 | V 64], 256 B) so one (candidate, head)
// stream is one contiguous byte range; each warp pulls its stream through a private 2-stage ring of 4 KB shared-memory
// buffers with TMA tensor loads + mbarrier (no registers held by loads in flight). The shared prompt prefix of the head
// is staged in shared memory once per CTA and reused by all of its candidates. At small batch several warps split one
// stream (flash-decoding) and merge through shared memory.
#include "common.cuh"
#include "ttb_internal.h"

#include <cstring>
#include <cstdio>
#include <vector>

namespace ttb {

constexpr int AS_THREADS = 512;
constexpr int AS_WARPS = AS_THREADS / 32;
constexpr int AS_CHUNK_POS = 16;                           // cache positions per ring stage
constexpr int AS_POS_BYTES = 256;                          // K row (64 bf16) + V row (64 bf16)
constexpr int AS_CHUNK_BYTES = AS_CHUNK_POS * AS_POS_BYTES;
constexpr int AS_RING_NS = 2;                              // ring stages per warp
constexpr int AS_RING_BYTES = AS_WARPS * AS_RING_NS * AS_CHUNK_BYTES;     // 128 KB
constexpr int AS_PREFIX_BYTES = 88 * 1024;
constexpr int AS_MAX_P = AS_PREFIX_BYTES / AS_POS_BYTES;         // 352 prompt positions
constexpr int AS_DATA_BYTES = AS_RING_BYTES + AS_PREFIX_BYTES;   // GEMM pipeline stages alias this region
constexpr int AS_CTRL_BYTES = 8 * 1024;
constexpr int AS_SMEM_TOTAL = AS_DATA_BYTES + AS_CTRL_BYTES + 1024;
constexpr int AS_MAX_STAGES = 8;
constexpr int AS_W_TILE_BYTES = 128 * 64 * 2;
constexpr int AS_MAX_TILES = 512;                          // ticket counters (row tile x batch tile)
constexpr int AS_SYNC_BAR_BYTES = 17 * 128;                // barrier epoch line + 16 arrival-counter lines
constexpr int AS_COMPACT_WARPS = 8;                        // ar_attn_compact_kernel: 256 threads, ~118 KB at P = 174
constexpr int AS_COMPACT_CTAS = 2;                         // ar_attn_compact_kernel CTAs per SM
constexpr int AS_MAX_GROUPS = 256;                         // prompt-prefix groups of one step (TtbArStepArgs.groups): one per row

enum { G_QKV = 0, G_PROJ = 1, G_FC = 2, G_PROJ2 = 3, G_HEAD = 4 };
enum { OUT_PARTIAL = 0, OUT_BF16 = 1, OUT_F32 = 2 };

struct AsGemmShape {
  int Nrows, K, KB, nsplit, kbps, n_rt, items, ldp;
};

struct AsLayer {       // device table, one per layer
  const float *ln1_g, *ln1_b, *bqkv, *bproj, *ln2_g, *ln2_b, *bfc, *bproj2;
};

// One prompt-prefix group of the attention phase: rows [b0, next b0) attend to a prefix of P positions (tensor map
// maps[4 L + 6 + g]); its attention units are [u0, next u0), ncph CTAs per head. Entry [groups] is a sentinel whose
// b0 is B and whose u0 is the total number of units. The table ([groups + 1] entries, up to 4 KB) lives in the device
// tables behind the layer table, not in the kernel parameters.
struct AsGroup {
  int b0, P, u0, ncph;
};

struct AsParams {
  int B, D, H, L, V, Nmax, pos_mode;
  int TB, nbt, nst, stage_bytes;          // batch tile (wgmma N), number of batch tiles, pipeline stages
  int units, ipr, team;                   // attention: work units (group, head, chunk), items per round, warps per item
  int ngroups;                            // prompt groups (1 when every row shares one prompt)
  int P0, ncph0;                          // prompt positions and CTAs per head of the batch when ngroups = 1
  int layer_begin, layer_end, phase_mask; // debug / profiling: subset of the step (phase_mask bit i = phase i of a layer)
  AsGemmShape g[5];
  const CUtensorMap* maps;                // device: [4*L + 1] weight maps, then activation maps a, o, h, hn
  const AsLayer* layers;                  // device: [L]
  const AsGroup* gtab;                    // device: [ngroups + 1], behind the layer table
  const float *lnf_g, *lnf_b, *fn_g, *fn_b, *b_head;
  const float *mel_emb, *mel_pos;
  const int* codes;
  int ld_codes;
  TtbArState* state;
  float* x;
  __nv_bfloat16 *a, *qkv, *o, *h, *hn;
  float* part;
  float* logits;
  const __nv_bfloat16* prefix_kv;         // [L][H][P][2][64] (group 0)
  __nv_bfloat16* cand_kv;                 // [L][B][H][Nmax][2][64]
  unsigned long long* bar;                // [0] barrier epoch at launch; arrival slots at [16 * (1 + k)], k < 16
  unsigned int* tickets;                  // [AS_MAX_TILES]
  int attn_data_bytes;                    // compact attention launch: rings of the active warps + the prompt of one head
  const int* row_start;                   // device [B] or NULL (TtbArStepArgs.row_start)
};

// Row b's own step: state->step without row_start, else step - row_start[b] clamped to [1, Nmax] (include/ttb.h), so
// that an idle row of a stream pool never indexes outside its codes and KV rows. ROWS = false compiles the row_start
// checks away: the launches without row_start (ar_step_kernel<false>, ar_attn_only_kernel<false>,
// ar_attn_compact_kernel<false>) are the kernels they were before row_start existed (a runtime branch in ar_step_kernel
// cost its one-row decode 1-2 % on H100).
template <bool ROWS>
TTB_DEVINL int row_step(const AsParams& p, int step, int b) {
  return (ROWS && p.row_start) ? min(max(step - __ldg(p.row_start + b), 1), p.Nmax) : step;
}

// phase bits (phase_mask)
enum { PH_EMBED = 1, PH_QKV = 2, PH_ATTN = 4, PH_PROJ = 8, PH_LN2 = 16, PH_FC = 32, PH_PROJ2 = 64, PH_LN1 = 128, PH_HEAD = 256,
       PH_NOP = 512 /* probe: one empty grid barrier per layer */ };

// ------------------------------------------------------------------ small device helpers
TTB_DEVINL void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }

TTB_DEVINL unsigned long long ld_acquire_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

TTB_DEVINL bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P1;\n\t"
#if TTB_MBAR_HINT_NS > 0
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2, %3;\n\t"    // parked up to the hint (common.cuh)
      "selp.u32 %0, 1, 0, P1;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"((uint32_t)TTB_MBAR_HINT_NS)
      : "memory");
#else
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P1;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
#endif
  return ok != 0;
}

// Bounded wait: a protocol error must end as an error flag, not as a hung GPU. ~2 s budget.
TTB_DEVINL void mbar_wait_to(uint64_t* bar, uint32_t parity, int* err) {
  if (mbar_try_wait(bar, parity)) return;
  unsigned long long t0 = 0;             // %globaltimer is slow to read: only once the wait is already long
  unsigned n = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++n & 0x3ff) == 0) {
      if (t0 == 0) t0 = global_timer_ns();
      if (*reinterpret_cast<volatile int*>(err) != 0) return;
      if (global_timer_ns() - t0 > 2000000000ull) { *reinterpret_cast<volatile int*>(err) = 2; return; }
    }
  }
}

TTB_DEVINL void tma_prefetch_3d(const CUtensorMap* map, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.prefetch.tensor.3d.L2.global.tile [%0, {%1, %2, %3}];" ::"l"(reinterpret_cast<uint64_t>(map)),
               "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}

TTB_DEVINL void named_bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

struct AsCtrl {                       // lives in the control block of shared memory
  uint64_t full_bar[AS_MAX_STAGES];
  uint64_t empty_bar[AS_MAX_STAGES];
  uint64_t ring_bar[AS_WARPS][AS_RING_NS];
  uint64_t prefix_bar;
  uint32_t ticket;
  float red[4][AS_WARPS];
  float merge[AS_WARPS][68];          // flash-decoding merge: acc[64], m, l
};
static_assert(sizeof(AsCtrl) <= AS_CTRL_BYTES, "control block too large");

struct AsCtrlCompact {                // control block of ar_attn_compact_kernel: only what the attention phase touches
  uint64_t ring_bar[AS_COMPACT_WARPS][AS_RING_NS];
  uint64_t prefix_bar;
  float merge[AS_COMPACT_WARPS][68];
};
constexpr int AS_CTRL_COMPACT_BYTES = (int)((sizeof(AsCtrlCompact) + 127) & ~size_t(127));

struct AsRole {                       // per-thread pipeline bookkeeping that survives across phases
  int stage;                          // GEMM smem ring position (producer and consumer threads keep identical copies)
  uint32_t phase;
  uint32_t ring_par[AS_RING_NS];      // attention ring parities of this warp
  uint32_t prefix_par;
  unsigned long long bar_target;      // next grid-barrier target
};

// ------------------------------------------------------------------ grid-wide barrier
// Arrivals are spread over AS_BAR_SLOTS counters, each on its own 128-byte line: one atomic per CTA on the same address serialises in one
// L2 slice; the first AS_BAR_SLOTS lanes of warp 0 poll one
// counter each. Counters are monotonic: slot k ends barrier number E at E * (number of CTAs mapped to slot k).
constexpr int AS_BAR_SLOTS = 16;
constexpr int AS_BAR_STRIDE = 16;          // u64 elements between slots (128 bytes)

TTB_DEVINL void grid_sync(const AsParams& p, AsRole& rl) {
  int* err = &p.state->reserved[0];
  // generic-proxy writes of this phase must be ordered before async-proxy (TMA) reads of later phases
  fence_proxy_async_all();
  __syncthreads();
  rl.bar_target += 1;                     // barrier epoch
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    if (lane == 0) {
      unsigned long long* slot = p.bar + AS_BAR_STRIDE * (1 + (blockIdx.x % AS_BAR_SLOTS));
      asm volatile("red.release.gpu.global.add.u64 [%0], 1;" ::"l"(slot) : "memory");
    }
    if (*reinterpret_cast<volatile int*>(err) == 0) {
      // CTAs mapped to slot `lane`: blockIdx % SLOTS == lane
      const unsigned long long cnt = (lane < AS_BAR_SLOTS) ? (gridDim.x + AS_BAR_SLOTS - 1 - lane) / AS_BAR_SLOTS : 0;
      const unsigned long long want = rl.bar_target * cnt;
      const unsigned long long* mine = p.bar + AS_BAR_STRIDE * (1 + (lane % AS_BAR_SLOTS));
      unsigned long long t0 = 0;
      unsigned n = 0;
      while (true) {
        const bool ok = (lane >= AS_BAR_SLOTS) || (ld_acquire_u64(mine) >= want);
        if (__all_sync(0xffffffffu, ok)) break;
        if ((++n & 0xff) == 0) {
          if (t0 == 0) t0 = global_timer_ns();
          const bool stop = (*reinterpret_cast<volatile int*>(err) != 0) || (global_timer_ns() - t0 > 2000000000ull);
          if (__any_sync(0xffffffffu, stop)) { if (lane == 0) *reinterpret_cast<volatile int*>(err) = 1; break; }
        }
      }
    }
  }
  __syncthreads();
}

// block-wide sum over 512 threads; `buf` is one of ctrl.red[i] (callers alternate buffers so one sync per reduction suffices)
TTB_DEVINL float block_sum16(float v, float* buf) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) buf[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < AS_WARPS; ++i) s += buf[i];
  return s;
}

// ------------------------------------------------------------------ L2 prefetch of the weight tiles this CTA will need
TTB_DEVINL void prefetch_gemm_item(const AsParams& p, const CUtensorMap* mw, const AsGemmShape& g) {
  for (int item = blockIdx.x; item < g.items; item += gridDim.x) {
    const int ks = item % g.nsplit;
    const int rt = (item / g.nsplit) / p.nbt;
    const int kb0 = ks * g.kbps;
    const int nkb = min(g.kbps, g.KB - kb0);
    for (int i = 0; i < nkb; ++i) tma_prefetch_3d(mw, (kb0 + i) * 64, rt * 128, 0);
  }
}

// ------------------------------------------------------------------ GEMM phase
// out[b, n] = act( sum_k act_in[b, k] * W[n, k] + bias[n] ),  n in [0, Nrows), b in [0, B)
template <int OUT, int ACT>
TTB_DEVINL void gemm_phase(const AsParams& p, const AsGemmShape& g, const CUtensorMap* mw, const CUtensorMap* ma,
                           const float* __restrict__ bias, void* out, int ldo, uint8_t* data, AsCtrl* ctrl, AsRole& rl) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int* err = &p.state->reserved[0];
  const int TB = p.TB;
  if (warp == 0) {
    // ===== TMA producer =====
    if (lane == 0) {
      for (int item = blockIdx.x; item < g.items; item += gridDim.x) {
        const int ks = item % g.nsplit;
        const int t = item / g.nsplit;
        const int bt = t % p.nbt, rt = t / p.nbt;
        const int kb0 = ks * g.kbps;
        const int nkb = min(g.kbps, g.KB - kb0);
        for (int i = 0; i < nkb; ++i) {
          mbar_wait_to(&ctrl->empty_bar[rl.stage], rl.phase ^ 1, err);
          uint8_t* sw = data + rl.stage * p.stage_bytes;
          uint8_t* sa = sw + AS_W_TILE_BYTES;
          mbar_arrive_expect_tx(&ctrl->full_bar[rl.stage], (uint32_t)p.stage_bytes);
          tma_load_3d(sw, mw, &ctrl->full_bar[rl.stage], (kb0 + i) * 64, rt * 128, 0);
          tma_load_3d(sa, ma, &ctrl->full_bar[rl.stage], (kb0 + i) * 64, bt * TB, 0);
          if (++rl.stage == p.nst) { rl.stage = 0; rl.phase ^= 1; }
        }
      }
    }
  } else if (warp >= 4) {
    // ===== warps 4..7 / 8..11: two consumer warpgroups (weight rows [0, 64) / [64, 128) of the tile; columns =
    //       candidates): wgmma main loop, then the epilogue straight from the accumulator fragments =====
    // ===== warps 12..15: idle during the main loop; they join the split-K fix-up of ticketed GEMMs (384 threads) =====
    const bool epi = warp < 12;
    const bool ticketed = (OUT != OUT_PARTIAL) && g.nsplit > 1;
    if (!epi && !ticketed) return;
    const int wg = (warp - 4) >> 2;
    const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);      // accumulator rows of this thread: row0, row0 + 8
    const int et = threadIdx.x - 128;                  // 0..383 (epilogue threads first)
    for (int item = blockIdx.x; item < g.items; item += gridDim.x) {
      const int ks = item % g.nsplit;
      const int t = item / g.nsplit;
      const int bt = t % p.nbt, rt = t / p.nbt;
      const int b_lo = bt * TB;
      if (epi) {
      const int kb0 = ks * g.kbps;
      const int nkb = min(g.kbps, g.KB - kb0);
      // the batch tile is TB = 16 nb16 columns wide: one m64n16k16 per 16 candidates (accumulator block j), 8 at most
      float acc[8][8];
      int prev = -1;
      for (int i = 0; i < nkb; ++i) {
        mbar_wait_to(&ctrl->full_bar[rl.stage], rl.phase, err);
        const uint32_t sw = smem_u32(data + rl.stage * p.stage_bytes) + wg * (64 * 128);
        const uint32_t sa = smem_u32(data + rl.stage * p.stage_bytes) + AS_W_TILE_BYTES;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint64_t dw = wgmma_desc_kmajor_sw128(sw + k * 32);
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (j * 16 < TB) wgmma_m64n16k16_bf16_ss(acc[j], dw, wgmma_desc_kmajor_sw128(sa + j * 2048 + k * 32), (i | k) != 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&ctrl->empty_bar[prev]);   // count 2: one arrive per warpgroup
        prev = rl.stage;
        if (++rl.stage == p.nst) { rl.stage = 0; rl.phase ^= 1; }
      }
      wgmma_wait<0>();
      if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&ctrl->empty_bar[prev]);
      const bool direct = (g.nsplit == 1) && (OUT != OUT_PARTIAL);
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int n = rt * 128 + row0 + 8 * hh;
        if (n >= g.Nrows) continue;
        const float bn = (direct && bias) ? __ldg(bias + n) : 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            const int c = j * 16 + 8 * (r >> 1) + 2 * (lane & 3) + (r & 1);
            const int b = b_lo + c;
            if (c < TB && b < p.B) {
              float v = acc[j][4 * (r >> 1) + 2 * hh + (r & 1)];
              if (direct) {
                v += bn;
                if (ACT == TTB_ACT_GELU_NEW) v = gelu_new(v);
                if (OUT == OUT_BF16) reinterpret_cast<__nv_bfloat16*>(out)[(long long)b * ldo + n] = __float2bfloat16(v);
                else reinterpret_cast<float*>(out)[(long long)b * ldo + n] = v;
              } else {
                p.part[((long long)ks * p.B + b) * g.ldp + n] = v;
              }
            }
          }
        }
      }
      }
      if (ticketed) {
        // ticket: the last split to arrive reduces the tile in split order (deterministic), adds bias, activates, writes
        if (epi) __threadfence();
        named_bar_sync(1, 384);
        const int tile = rt * p.nbt + bt;
        if (et == 0) ctrl->ticket = atomicAdd(&p.tickets[tile], 1u);
        named_bar_sync(1, 384);
        const bool last = (ctrl->ticket == (uint32_t)(g.nsplit - 1));
        named_bar_sync(1, 384);                          // ticket slot may be rewritten by the next item
        if (last) {
          __threadfence();
          const int nb = min(TB, p.B - b_lo);
          const int c4 = (et & 31) * 4;                  // 4 consecutive weight rows
          const int n4 = rt * 128 + c4;
          if (n4 < g.Nrows) {
            float4 bb = make_float4(0.f, 0.f, 0.f, 0.f);
            if (bias) {
              bb.x = __ldg(bias + n4);
              if (n4 + 1 < g.Nrows) bb.y = __ldg(bias + n4 + 1);
              if (n4 + 2 < g.Nrows) bb.z = __ldg(bias + n4 + 2);
              if (n4 + 3 < g.Nrows) bb.w = __ldg(bias + n4 + 3);
            }
            // 4 rows x all splits in flight per thread before the first add (a dependent chain of L2 round trips
            // otherwise dominates this fix-up)
            constexpr int FX_ROWS = 2, FX_SPLITS = 4, FX_LANES = 12;      // 384 threads = 32 column groups x 12 row lanes
            for (int bi0 = (et >> 5); bi0 < nb; bi0 += FX_LANES * FX_ROWS) {
              float4 acc[FX_ROWS];
#pragma unroll
              for (int r = 0; r < FX_ROWS; ++r) acc[r] = bb;
              for (int sp0 = 0; sp0 < g.nsplit; sp0 += FX_SPLITS) {
                float4 v[FX_ROWS][FX_SPLITS];
#pragma unroll
                for (int r = 0; r < FX_ROWS; ++r) {
                  const int bi = bi0 + FX_LANES * r;
#pragma unroll
                  for (int u = 0; u < FX_SPLITS; ++u) {
                    v[r][u] = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (bi < nb && sp0 + u < g.nsplit)
                      v[r][u] = __ldcg(reinterpret_cast<const float4*>(p.part + ((long long)(sp0 + u) * p.B + b_lo + bi) * g.ldp + n4));
                  }
                }
#pragma unroll
                for (int r = 0; r < FX_ROWS; ++r)
#pragma unroll
                  for (int u = 0; u < FX_SPLITS; ++u) {       // fixed split order: deterministic
                    acc[r].x += v[r][u].x; acc[r].y += v[r][u].y; acc[r].z += v[r][u].z; acc[r].w += v[r][u].w;
                  }
              }
#pragma unroll
              for (int r = 0; r < FX_ROWS; ++r) {
                const int bi = bi0 + FX_LANES * r;
                if (bi >= nb) continue;
                const int b = b_lo + bi;
                float4 s = acc[r];
                if (ACT == TTB_ACT_GELU_NEW) { s.x = gelu_new(s.x); s.y = gelu_new(s.y); s.z = gelu_new(s.z); s.w = gelu_new(s.w); }
                if (OUT == OUT_BF16) {
                  __nv_bfloat16* op = reinterpret_cast<__nv_bfloat16*>(out) + (long long)b * ldo + n4;
                  if (n4 + 3 < g.Nrows && (ldo & 3) == 0) {
                    *reinterpret_cast<uint2*>(op) = make_uint2(pack_bf16(s.x, s.y), pack_bf16(s.z, s.w));
                  } else {
                    op[0] = __float2bfloat16(s.x);
                    if (n4 + 1 < g.Nrows) op[1] = __float2bfloat16(s.y);
                    if (n4 + 2 < g.Nrows) op[2] = __float2bfloat16(s.z);
                    if (n4 + 3 < g.Nrows) op[3] = __float2bfloat16(s.w);
                  }
                } else {
                  float* op = reinterpret_cast<float*>(out) + (long long)b * ldo + n4;
                  op[0] = s.x;
                  if (n4 + 1 < g.Nrows) op[1] = s.y;
                  if (n4 + 2 < g.Nrows) op[2] = s.z;
                  if (n4 + 3 < g.Nrows) op[3] = s.w;
                }
              }
            }
          }
          if (et == 0) p.tickets[tile] = 0;
        }
      }
    }
  }
}

// ------------------------------------------------------------------ attention phase
// A SIMT form spends ~14 issue slots per cached position (bf16 unpacking, 8-lane dot products, shuffles): at 256
// candidates it is issue-bound rather than bound by its KV traffic, and the shared prompt part is a large share of it.
// Here both products of a 16-position chunk run on the tensor cores (mma.sync m16n8k16, bf16 in / fp32 out):
//   S[16 pos] = K[16 x 64] q      : A = K chunk (row = position), B = q in column 0 of the 16 x 8 operand
//   O[64]    += V^T[64 x 16] p    : A = V chunk read transposed (ldmatrix.trans), B = p (bf16) in column 0
// 7/8 of every MMA is padding - the tensor pipe is idle anyway, what matters is ~3 issue slots per position.
// K and V rows are separate 2 KB tiles in shared memory, written by TMA with the 128-byte swizzle, so that the eight
// 16-byte rows of an ldmatrix fall into distinct banks (the 256-byte position pitch of the raw cache would alias them).
TTB_DEVINL void tma_load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
TTB_DEVINL void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
TTB_DEVINL void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
TTB_DEVINL void mma_bf16_16816(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

struct MmaState {
  float m;             // running max (log2 domain), warp-uniform
  float l;             // this lane's share of the running sum
  float acc[4][4];     // O^T accumulators: dim block db, fragment regs; column 0 lives in lanes with lane % 4 == 0:
                       //   acc[db][0] = O[16 db + lane/4], acc[db][2] = O[16 db + lane/4 + 8]
};

// one chunk: K tile / V tile (16 rows x 128 B, SWIZZLE_128B) at shared addresses kt / vt, npos valid rows
TTB_DEVINL void mma_chunk(MmaState& st, const uint32_t* qb, uint32_t kt, uint32_t vt, int npos, int lane) {
  const int mi = lane >> 3, r = lane & 7;
  const int pos = r + 8 * (mi & 1);                       // row this lane addresses for K (matrices 0/1: rows 0-7 / 8-15)
  float s[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    uint32_t a0, a1, a2, a3;
    const int ch = ks * 2 + (mi >> 1);                    // 16-byte chunk (8 dims) inside the 128-byte row
    ldsm_x4(kt + pos * 128 + ((ch ^ (pos & 7)) << 4), a0, a1, a2, a3);
    mma_bf16_16816(s, a0, a1, a2, a3, qb[2 * ks], qb[2 * ks + 1]);
  }
  const bool act = (lane & 3) == 0;
  const int j = lane >> 2;
  const float sc = 0.125f * 1.4426950408889634f;          // 1/sqrt(64) and log2(e)
  float s_lo = (act && j < npos) ? s[0] * sc : -INFINITY;
  float s_hi = (act && j + 8 < npos) ? s[2] * sc : -INFINITY;
  float mx = fmaxf(s_lo, s_hi);
  mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 4));
  mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 8));
  mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 16));
  const float m_new = fmaxf(st.m, mx);
  const float m_use = (m_new == -INFINITY) ? 0.f : m_new;
  const float corr = exp2f(st.m - m_use);
  st.m = m_new;
  const float p_lo = exp2f(s_lo - m_use), p_hi = exp2f(s_hi - m_use);
  st.l = st.l * corr + p_lo + p_hi;
  // p as the B operand (k = position, column 0): lanes 0-3 need p[2l], p[2l+1], p[2l+8], p[2l+9]
  const int src = 8 * (lane & 3);
  const float x0 = __shfl_sync(0xffffffffu, p_lo, src), x1 = __shfl_sync(0xffffffffu, p_lo, src + 4);
  const float y0 = __shfl_sync(0xffffffffu, p_hi, src), y1 = __shfl_sync(0xffffffffu, p_hi, src + 4);
  const uint32_t b0 = (lane < 4) ? pack_bf16(x0, x1) : 0u;
  const uint32_t b1 = (lane < 4) ? pack_bf16(y0, y1) : 0u;
  const int vpos = r + 8 * (mi >> 1);                     // V (transposed read): matrices 0/1 rows 0-7, 2/3 rows 8-15
#pragma unroll
  for (int db = 0; db < 4; ++db) {
#pragma unroll
    for (int i = 0; i < 4; ++i) st.acc[db][i] *= corr;
    uint32_t a0, a1, a2, a3;
    const int ch = db * 2 + (mi & 1);
    ldsm_x4_t(vt + vpos * 128 + ((ch ^ (vpos & 7)) << 4), a0, a1, a2, a3);
    mma_bf16_16816(st.acc[db], a0, a1, a2, a3, b0, b1);
  }
}

// `wait_pdl`: the caller has NOT yet executed griddepcontrol.wait (ar_attn_only_kernel under programmatic dependent
// launch): the prompt prefix and the first candidate tiles are requested first -- the caches were written by earlier
// steps / this step's earlier kernels, only q and the new K / V come from the c_attn GEMM this launch depends on.
template <bool ROWS, class CtrlT>
TTB_DEVINL void attn_phase_mma(const AsParams& p, int layer, uint8_t* data, CtrlT* ctrl, AsRole& rl, bool wait_pdl = false) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int* err = &p.state->reserved[0];
  const int B = p.B, H = p.H, Nmax = p.Nmax, D = p.H * 64;
  constexpr int NS = AS_RING_NS;
  constexpr int CHUNK_BYTES = AS_CHUNK_BYTES;          // K tile 2 KB | V tile 2 KB
  const int step = p.state->step;
  const int slot0 = step - 1;                          // KV slot and candidate length of every row without row_start
  uint8_t* ring = data + warp * NS * CHUNK_BYTES;
  uint8_t* prefix_s = data + p.ipr * p.team * NS * CHUNK_BYTES;   // behind the rings of the active warps (host checks the fit)
  const CUtensorMap* map_c = p.maps + 4 * p.L + 5;
  __nv_bfloat16* ckv_l = p.cand_kv + (long long)layer * B * H * Nmax * 128;
  int g = 0;
  for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
    // the unit's group: the last g with u0 <= u, by bisection over [g, ngroups) (a CTA's units only grow, so its group
    // only advances). One group (every tts() call): the values come from the parameters; reading the table here cost
    // ~2 % of the one-row decode of 603 tokens on H100. With row_start the table is read even for one group: a stream
    // pool rewrites its groups' P between steps (ttb_ar_step_set_group_len)
    int gb0 = 0, gB = B, ncph = p.ncph0, P = p.P0, lu = u;
    if (p.ngroups > 1 || (ROWS && p.row_start)) {
      for (int hi = p.ngroups; hi - g > 1;) {
        const int mid = (g + hi) >> 1;
        if (__ldg(&p.gtab[mid].u0) <= u) g = mid; else hi = mid;
      }
      const AsGroup* ge = p.gtab + g;
      gb0 = __ldg(&ge->b0); gB = __ldg(&ge[1].b0) - gb0; ncph = __ldg(&ge->ncph);
      P = __ldg(&ge->P);
      lu = u - __ldg(&ge->u0);
    }
    const CUtensorMap* map_p = map_c + 1 + g;            // prompt prefix of this unit's group
    const int npc = (P + 15) / 16;
    const int h = lu % H, ci = lu / H;
    const int b_begin = gb0 + (int)((long long)ci * gB / ncph), b_end = gb0 + (int)((long long)(ci + 1) * gB / ncph);
    __syncthreads();
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(&ctrl->prefix_bar, (uint32_t)(npc * CHUNK_BYTES));
      for (int c = 0; c < npc; ++c) {
        tma_load_4d(prefix_s + c * CHUNK_BYTES, map_p, &ctrl->prefix_bar, 0, 0, c * 16, layer * H + h);
        tma_load_4d(prefix_s + c * CHUNK_BYTES + 2048, map_p, &ctrl->prefix_bar, 0, 1, c * 16, layer * H + h);
      }
    }
    const int sub = warp % p.team;
    const int nch0 = (slot0 + 15) / 16;
    // first NS tiles of candidate bb's stream into this warp's ring (lane 0). All stages are free whenever this is
    // called: at the start of the unit, or after the last tile of the previous item was consumed.
    auto issue_head = [&](int bb) {
      const int it = (layer * B + bb) * H + h;
      const int nch = ROWS ? (row_step<ROWS>(p, step, bb) - 1 + 15) / 16 : nch0;   // chunks of bb's own length
      for (int s = 0; s < NS; ++s) {
        const int c = sub + s * p.team;
        if (c < nch) {
          mbar_arrive_expect_tx(&ctrl->ring_bar[warp][s], (uint32_t)CHUNK_BYTES);
          tma_load_4d(ring + s * CHUNK_BYTES, map_c, &ctrl->ring_bar[warp][s], 0, 0, c * 16, it);
          tma_load_4d(ring + s * CHUNK_BYTES + 2048, map_c, &ctrl->ring_bar[warp][s], 0, 1, c * 16, it);
        }
      }
    };
    bool head_issued = false;        // the stream of this round's item was started during the previous round
    for (int r0 = b_begin; r0 < b_end; r0 += p.ipr) {
      const int b = r0 + warp / p.team;
      const bool valid = (warp < p.ipr * p.team) && (b < b_end);
      MmaState st;
      st.m = -INFINITY; st.l = 0.f;
#pragma unroll
      for (int db = 0; db < 4; ++db)
#pragma unroll
        for (int i = 0; i < 4; ++i) st.acc[db][i] = 0.f;
      // the KV stream first (it needs addresses only), then q: the q loads overlap the first tiles' latency
      if (valid && !head_issued && lane == 0) issue_head(b);
      if (wait_pdl) { pdl_wait(); wait_pdl = false; }
      if (valid) {
        const int slot = ROWS ? row_step<ROWS>(p, step, b) - 1 : slot0;   // KV slot written = positions before it
        const int nold = slot;
        const int nch = ROWS ? (nold + 15) / 16 : nch0;
        const __nv_bfloat16* qrow = p.qkv + (long long)b * 3 * D + h * 64;
        // q as the B operand of the score MMA: column 0 <-> lanes 0-3; b0 = dims 16 ks + 2 lane (+1), b1 = + 8
        uint32_t qb[8];
        const uint32_t* q32 = reinterpret_cast<const uint32_t*>(qrow);
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          qb[2 * ks] = (lane < 4) ? __ldcg(q32 + ks * 8 + lane) : 0u;
          qb[2 * ks + 1] = (lane < 4) ? __ldcg(q32 + ks * 8 + 4 + lane) : 0u;
        }
        __nv_bfloat16* cb = ckv_l + ((long long)b * H + h) * Nmax * 128;
        const int item = (layer * B + b) * H + h;          // 4th coordinate of the candidate-cache tensor map
        if (sub == 0) {
          // the new token: append K / V to the cache, account for it from registers (SIMT, once per item)
          const uint32_t kq = __ldcg(reinterpret_cast<const uint32_t*>(qrow + D) + lane);      // dims 2 lane, 2 lane + 1
          const uint32_t qq = __ldcg(q32 + lane);
          const float2 kf = unpack_bf16(kq), qf = unpack_bf16(qq);
          float sn = warp_sum(kf.x * qf.x + kf.y * qf.y) * (0.125f * 1.4426950408889634f);
          if (lane < 16) {
            const uint4 nv = __ldcg(reinterpret_cast<const uint4*>(qrow + (lane < 8 ? D : 2 * D)) + (lane & 7));
            reinterpret_cast<uint4*>(cb + (long long)slot * 128 + (lane < 8 ? 0 : 64))[lane & 7] = nv;
          }
          st.m = sn;
          st.l = (lane == 0) ? 1.f : 0.f;
          if ((lane & 3) == 0) {
            const __nv_bfloat16* vrow = qrow + 2 * D;
            const int j = lane >> 2;
#pragma unroll
            for (int db = 0; db < 4; ++db) {
              st.acc[db][0] = __bfloat162float(vrow[db * 16 + j]);
              st.acc[db][2] = __bfloat162float(vrow[db * 16 + j + 8]);
            }
          }
        }
        int s = 0;
        // The prompt part (npc chunks already in shared memory, the same for every candidate of this head) is worked
        // off one chunk at a time BEFORE each wait for a candidate tile: the warp would otherwise sit idle at the ring
        // barrier (a tile takes several times longer to arrive than a chunk takes to compute), and doing the prompt part after
        // the stream leaves the memory system idle once per round.
        int pc = sub;
        bool prefix_ready = false;
        for (int c_use = sub; c_use < nch; c_use += p.team) {
          if (pc < npc) {
            if (!prefix_ready) { mbar_wait_to(&ctrl->prefix_bar, rl.prefix_par, err); prefix_ready = true; }
            const uint32_t kp = smem_u32(prefix_s + pc * CHUNK_BYTES);
            mma_chunk(st, qb, kp, kp + 2048, min(16, P - pc * 16), lane);
            pc += p.team;
          }
          mbar_wait_to(&ctrl->ring_bar[warp][s], rl.ring_par[s], err);
          rl.ring_par[s] ^= 1;
          const uint32_t kt = smem_u32(ring + s * CHUNK_BYTES);
          mma_chunk(st, qb, kt, kt + 2048, min(16, nold - c_use * 16), lane);
          __syncwarp();
          const int c_next = c_use + NS * p.team;
          if (lane == 0 && c_next < nch) {
            mbar_arrive_expect_tx(&ctrl->ring_bar[warp][s], (uint32_t)CHUNK_BYTES);
            tma_load_4d(ring + s * CHUNK_BYTES, map_c, &ctrl->ring_bar[warp][s], 0, 0, c_next * 16, item);
            tma_load_4d(ring + s * CHUNK_BYTES + 2048, map_c, &ctrl->ring_bar[warp][s], 0, 1, c_next * 16, item);
          }
          if (++s == NS) s = 0;
        }
        // every stage is free again: start the stream of this warp's NEXT item now, so that its first tiles travel
        // while the prompt part, the merge and the output of this item are computed (the rounds of all warps and SMs
        // run in step: without this the memory system idles once per round)
        head_issued = (b + p.ipr < b_end);
        if (head_issued && lane == 0) issue_head(b + p.ipr);
        if (!prefix_ready) mbar_wait_to(&ctrl->prefix_bar, rl.prefix_par, err);
        for (int c = pc; c < npc; c += p.team) {             // what is left of the prompt part (long prompts, early steps)
          const uint32_t kt = smem_u32(prefix_s + c * CHUNK_BYTES);
          mma_chunk(st, qb, kt, kt + 2048, min(16, P - c * 16), lane);
        }
        st.l = warp_sum(st.l);
      }
      // ---- gather the row: (m, l, O[64]) of this warp into the scratch; leaders merge the team and write o
      float* ms = ctrl->merge[warp];
      if (valid) {
        if ((lane & 3) == 0) {
          const int j = lane >> 2;
#pragma unroll
          for (int db = 0; db < 4; ++db) { ms[db * 16 + j] = st.acc[db][0]; ms[db * 16 + j + 8] = st.acc[db][2]; }
        }
        if (lane == 0) { ms[64] = st.m; ms[65] = st.l; }
      }
      if (p.team > 1) __syncthreads(); else __syncwarp();
      if (valid && sub == 0 && lane < 8) {
        float m = ms[64], l = ms[65];
        float o[8];
#pragma unroll
        for (int d = 0; d < 8; ++d) o[d] = ms[lane * 8 + d];
        for (int t = 1; t < p.team; ++t) {
          const float* mo = ctrl->merge[warp + t];
          const float m_o = mo[64], l_o = mo[65];
          const float m_new = fmaxf(m, m_o);
          const float m_use = (m_new == -INFINITY) ? 0.f : m_new;
          const float c_s = exp2f(m - m_use), c_o = exp2f(m_o - m_use);
          l = l * c_s + l_o * c_o;
#pragma unroll
          for (int d = 0; d < 8; ++d) o[d] = o[d] * c_s + mo[lane * 8 + d] * c_o;
          m = m_new;
        }
        const float inv = 1.0f / l;
        reinterpret_cast<uint4*>(p.o + (long long)b * D + h * 64)[lane] =
            make_uint4(pack_bf16(o[0] * inv, o[1] * inv), pack_bf16(o[2] * inv, o[3] * inv),
                       pack_bf16(o[4] * inv, o[5] * inv), pack_bf16(o[6] * inv, o[7] * inv));
      }
      if (p.team > 1) __syncthreads(); else __syncwarp();     // scratch is rewritten by the next round
    }
    rl.prefix_par ^= 1;
  }
}

// ------------------------------------------------------------------ LayerNorm phases (one row per CTA pass, 512 threads)
// mode 0: x = mel_emb[tok] + mel_pos[pos]        (ar_embed_step)
// mode 1: x += rbias + sum_s part[s]             (residual update folded with the split-K reduction)
// then y = LN(x; g1, b1) [-> LN(.; g2, b2)] -> bf16 out
template <bool ROWS>
TTB_DEVINL void ln_phase(const AsParams& p, int mode, const float* part, int nsplit, int ldp, const float* __restrict__ rbias,
                         const float* __restrict__ g1, const float* __restrict__ b1, const float* __restrict__ g2,
                         const float* __restrict__ b2, __nv_bfloat16* out, AsCtrl* ctrl) {
  const int D = p.D;
  const int t = threadIdx.x;
  int rb = 0;
  for (int row = blockIdx.x; row < p.B; row += gridDim.x) {
    float v[2];
    if (mode == 0) {
      const int j = row_step<ROWS>(p, p.state->step, row);
      const int tok = p.codes[(long long)row * p.ld_codes + j - 1];
      const int pos = p.pos_mode ? j + 1 : j;          // autoregressive.py:147-149 (SURVEY App. D-1)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int c = t + i * AS_THREADS;
        v[i] = (c < D) ? __ldg(p.mel_emb + (long long)tok * D + c) + __ldg(p.mel_pos + (long long)pos * D + c) : 0.f;
      }
    } else {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int c = t + i * AS_THREADS;
        float a = 0.f;
        if (c < D) {
          float acc = rbias ? __ldg(rbias + c) : 0.f;
          const float xv = __ldcg(p.x + (long long)row * D + c);
          for (int sp0 = 0; sp0 < nsplit; sp0 += 8) {          // all loads first, then the adds in split order
            float pv[8];
#pragma unroll
            for (int u = 0; u < 8; ++u)
              pv[u] = (sp0 + u < nsplit) ? __ldcg(part + ((long long)(sp0 + u) * p.B + row) * ldp + c) : 0.f;
#pragma unroll
            for (int u = 0; u < 8; ++u) acc += pv[u];
          }
          a = xv + acc;
        }
        v[i] = a;
      }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int c = t + i * AS_THREADS;
      if (c < D) p.x[(long long)row * D + c] = v[i];
    }
#pragma unroll
    for (int pass = 0; pass < 2; ++pass) {
      const float* gg = pass == 0 ? g1 : g2;
      const float* bb = pass == 0 ? b1 : b2;
      if (!gg) break;
      const float mean = block_sum16(v[0] + v[1], ctrl->red[rb]) / D;
      rb = (rb + 1) & 3;
      float qs = 0.f;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int c = t + i * AS_THREADS;
        const float dx = (c < D) ? v[i] - mean : 0.f;
        qs += dx * dx;
      }
      const float rstd = rsqrtf(block_sum16(qs, ctrl->red[rb]) / D + 1e-5f);
      rb = (rb + 1) & 3;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int c = t + i * AS_THREADS;
        if (c < D) v[i] = (v[i] - mean) * rstd * __ldg(gg + c) + __ldg(bb + c);
      }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int c = t + i * AS_THREADS;
      if (c < D) out[(long long)row * D + c] = __float2bfloat16(v[i]);
    }
  }
}

// ------------------------------------------------------------------ the step kernel
template <bool ROWS>
__global__ void __launch_bounds__(AS_THREADS, 1) ar_step_kernel(const __grid_constant__ AsParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* data = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  AsCtrl* ctrl = reinterpret_cast<AsCtrl*>(data + AS_DATA_BYTES);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    for (int s = 0; s < AS_MAX_STAGES; ++s) { mbar_init(&ctrl->full_bar[s], 1); mbar_init(&ctrl->empty_bar[s], 2); }
    for (int w = 0; w < AS_WARPS; ++w)
      for (int k = 0; k < AS_RING_NS; ++k) mbar_init(&ctrl->ring_bar[w][k], 1);
    mbar_init(&ctrl->prefix_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  AsRole rl;
  rl.stage = 0; rl.phase = 0; rl.prefix_par = 0;
  rl.ring_par[0] = rl.ring_par[1] = 0;
  rl.bar_target = ld_acquire_u64(p.bar);          // barrier epoch at launch (bar[0]; the arrival slots follow)

  const CUtensorMap* map_a = p.maps + 4 * p.L + 1;
  const CUtensorMap* map_o = map_a + 1;
  const CUtensorMap* map_h = map_a + 2;
  const CUtensorMap* map_hn = map_a + 3;
  const bool pf = warp == 2 && lane == 0;            // L2 prefetch of the next phases' weight tiles
  const int L0 = p.layer_begin, L1 = p.layer_end;
  // the barrier behind the last phase of the launch orders nothing (the kernel boundary does): skip it
  int last_bit = 0;
  for (int b = 0; b < 10; ++b) if (p.phase_mask & (1 << b)) last_bit = b;
  const bool head_follows = (p.phase_mask & PH_HEAD) != 0;
#define AS_SYNC_UNLESS_LAST(bit, layer) \
  do { if (head_follows || (layer) + 1 < L1 || (bit) != last_bit) grid_sync(p, rl); } while (0)

  if (p.phase_mask & PH_EMBED) {
    if (pf && L0 < L1) prefetch_gemm_item(p, p.maps + 4 * L0 + G_QKV, p.g[G_QKV]);
    const AsLayer& l0 = p.layers[L0 < p.L ? L0 : 0];
    ln_phase<ROWS>(p, 0, nullptr, 0, 0, nullptr, l0.ln1_g, l0.ln1_b, nullptr, nullptr, p.a, ctrl);
    grid_sync(p, rl);
  }
  for (int l = L0; l < L1; ++l) {
    const AsLayer& lw = p.layers[l];
    const CUtensorMap* mw = p.maps + 4 * l;
    if (p.phase_mask & PH_QKV) {
      if (pf) { prefetch_gemm_item(p, mw + G_PROJ, p.g[G_PROJ]); prefetch_gemm_item(p, mw + G_FC, p.g[G_FC]); }
      gemm_phase<OUT_BF16, TTB_ACT_NONE>(p, p.g[G_QKV], mw + G_QKV, map_a, lw.bqkv, p.qkv, 3 * p.D, data, ctrl, rl);
      AS_SYNC_UNLESS_LAST(1, l);
    }
    if (p.phase_mask & PH_ATTN) {
      attn_phase_mma<ROWS>(p, l, data, ctrl, rl);
      AS_SYNC_UNLESS_LAST(2, l);
    }
    if (p.phase_mask & PH_NOP) grid_sync(p, rl);
    if (p.phase_mask & PH_PROJ) {
      if (pf) prefetch_gemm_item(p, mw + G_PROJ2, p.g[G_PROJ2]);
      gemm_phase<OUT_PARTIAL, TTB_ACT_NONE>(p, p.g[G_PROJ], mw + G_PROJ, map_o, nullptr, nullptr, 0, data, ctrl, rl);
      AS_SYNC_UNLESS_LAST(3, l);
    }
    if (p.phase_mask & PH_LN2) {
      ln_phase<ROWS>(p, 1, p.part, p.g[G_PROJ].nsplit, p.g[G_PROJ].ldp, lw.bproj, lw.ln2_g, lw.ln2_b, nullptr, nullptr, p.a, ctrl);
      AS_SYNC_UNLESS_LAST(4, l);
    }
    if (p.phase_mask & PH_FC) {
      if (pf) {
        if (l + 1 < p.L) prefetch_gemm_item(p, mw + 4 + G_QKV, p.g[G_QKV]);
        else prefetch_gemm_item(p, p.maps + 4 * p.L, p.g[G_HEAD]);
      }
      gemm_phase<OUT_BF16, TTB_ACT_GELU_NEW>(p, p.g[G_FC], mw + G_FC, map_a, lw.bfc, p.h, 4 * p.D, data, ctrl, rl);
      AS_SYNC_UNLESS_LAST(5, l);
    }
    if (p.phase_mask & PH_PROJ2) {
      gemm_phase<OUT_PARTIAL, TTB_ACT_NONE>(p, p.g[G_PROJ2], mw + G_PROJ2, map_h, nullptr, nullptr, 0, data, ctrl, rl);
      AS_SYNC_UNLESS_LAST(6, l);
    }
    if (p.phase_mask & PH_LN1) {
      if (l + 1 < p.L) {
        const AsLayer& nx = p.layers[l + 1];
        ln_phase<ROWS>(p, 1, p.part, p.g[G_PROJ2].nsplit, p.g[G_PROJ2].ldp, lw.bproj2, nx.ln1_g, nx.ln1_b, nullptr, nullptr, p.a, ctrl);
      } else {
        ln_phase<ROWS>(p, 1, p.part, p.g[G_PROJ2].nsplit, p.g[G_PROJ2].ldp, lw.bproj2, p.lnf_g, p.lnf_b, p.fn_g, p.fn_b, p.hn, ctrl);
      }
      AS_SYNC_UNLESS_LAST(7, l);
    }
  }
  if (p.phase_mask & PH_HEAD) {
    gemm_phase<OUT_F32, TTB_ACT_NONE>(p, p.g[G_HEAD], p.maps + 4 * p.L, map_hn, p.b_head, p.logits, p.V, data, ctrl, rl);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    // every CTA has read the epoch before its first arrival, and all arrivals of this launch precede this point
    *reinterpret_cast<volatile unsigned long long*>(p.bar) = rl.bar_target;
  }
}

// The attention phase alone as an ordinary (non-cooperative) launch: no grid barrier. Used by the "mixed" decode
// mode, where the GEMMs / LayerNorms of the step stay separate kernels (see ar_engine.py).
template <bool ROWS>
__global__ void __launch_bounds__(AS_THREADS, 1) ar_attn_only_kernel(const __grid_constant__ AsParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* data = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  AsCtrl* ctrl = reinterpret_cast<AsCtrl*>(data + AS_DATA_BYTES);
  if (threadIdx.x == 0) {
    for (int w = 0; w < AS_WARPS; ++w)
      for (int k = 0; k < AS_RING_NS; ++k) mbar_init(&ctrl->ring_bar[w][k], 1);
    mbar_init(&ctrl->prefix_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  AsRole rl;
  rl.stage = 0; rl.phase = 0; rl.prefix_par = 0; rl.bar_target = 0;
  rl.ring_par[0] = rl.ring_par[1] = 0;
  attn_phase_mma<ROWS>(p, p.layer_begin, data, ctrl, rl, true);   // waits for the c_attn GEMM (PDL) after its first requests
  pdl_launch_dependents();
}

// The same phase in a CTA that leaves half of the SM free (TtbArStepArgs.attn_compact): 8 warps, shared memory = the
// rings of the active warps + the prompt of ONE head + a small control block (111.5 KB at P = 174 instead of 225 KB), so
// that a skinny-GEMM CTA (101 KB, 192 threads) of ANOTHER decode chain fits beside it -- or a second CTA of this kernel
// (prompts up to 176 positions), which gives the SM its 16 concurrent KV streams back when the kernel has it to itself. Used when the candidates are decoded
// as two independent half-batches on two streams (ar_engine.py, TTB_AR_CHAINS): the latency-bound GEMM / LayerNorm
// chain of one half then overlaps the bandwidth-bound attention of the other.
template <bool ROWS>
__global__ void __launch_bounds__(AS_COMPACT_WARPS * 32, AS_COMPACT_CTAS) ar_attn_compact_kernel(const __grid_constant__ AsParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* data = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  AsCtrlCompact* ctrl = reinterpret_cast<AsCtrlCompact*>(data + p.attn_data_bytes);
  if (threadIdx.x == 0) {
    for (int w = 0; w < AS_COMPACT_WARPS; ++w)
      for (int k = 0; k < AS_RING_NS; ++k) mbar_init(&ctrl->ring_bar[w][k], 1);
    mbar_init(&ctrl->prefix_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  AsRole rl;
  rl.stage = 0; rl.phase = 0; rl.prefix_par = 0; rl.bar_target = 0;
  rl.ring_par[0] = rl.ring_par[1] = 0;
  attn_phase_mma<ROWS>(p, p.layer_begin, data, ctrl, rl, true);
  pdl_launch_dependents();
}

// prompt K/V from a qkv buffer [P, 3*H*64] into the interleaved prefix cache [H][cap][K 64 | V 64] (cap >= P positions
// per head: a stream pool's slot buffers are sized for the longest prompt)
__global__ void ar_step_store_prefix_kernel(const __nv_bfloat16* __restrict__ qkv, int P, int cap, int H,
                                            __nv_bfloat16* __restrict__ pkv) {
  const int D = H * 64;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // over P * D
  if (i >= (long long)P * D) return;
  const int pp = (int)(i / D), c = (int)(i - (long long)pp * D);
  const int h = c >> 6, d = c & 63;
  __nv_bfloat16* dst = pkv + ((long long)h * cap + pp) * 128;
  dst[d] = qkv[(long long)pp * 3 * D + D + c];
  dst[64 + d] = qkv[(long long)pp * 3 * D + 2 * D + c];
}

// one group's prompt length in the device group table (ttb_ar_step_set_group_len); stream-ordered, graph-free
__global__ void ar_step_set_group_len_kernel(AsGroup* gtab, int g, int P) { gtab[g].P = P; }

// ------------------------------------------------------------------ host: plan
struct AsPlan {
  AsParams p;
  AsGroup gtab[AS_MAX_GROUPS + 1];        // host copy of the group table (ttb_ar_step_setup writes it to the device)
  long long part_floats;
  int grid;
  int ngroups;                            // >= 1 (groups == 0 is one group of every row)
};

static int as_num_sms() {
  int dev = 0, n = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  return n > 0 ? n : 132;
}

static int env_int(const char* name, int dflt) {
  const char* e = getenv(name);
  return e ? atoi(e) : dflt;
}

static void plan_gemm(AsGemmShape& g, int Nrows, int K, int nbt, int grid, int cap) {
  g.Nrows = Nrows; g.K = K; g.KB = K / 64;
  g.n_rt = (Nrows + 127) / 128;
  g.ldp = (Nrows + 3) & ~3;
  int ns = grid / (g.n_rt * nbt);
  if (ns < 1) ns = 1;
  if (ns > cap) ns = cap;
  if (ns > g.KB) ns = g.KB;
  g.kbps = (g.KB + ns - 1) / ns;
  g.nsplit = (g.KB + g.kbps - 1) / g.kbps;
  g.items = g.n_rt * nbt * g.nsplit;
}

static int make_plan(const TtbArStepArgs& a, AsPlan& pl) {
  AsParams& p = pl.p;
  memset(&p, 0, sizeof(p));
  memset(pl.gtab, 0, sizeof(pl.gtab));
  if (a.B <= 0 || a.B > 256) { set_error("ttb_ar_step: B=%d unsupported (1..256)", a.B); return -1; }
  if (a.D != a.H * 64 || a.D % 128 != 0 || a.D > 1024) { set_error("ttb_ar_step: D=%d H=%d unsupported (D = 64 H, D %% 128 == 0, D <= 1024)", a.D, a.H); return -1; }
  if (a.groups < 0 || a.groups > AS_MAX_GROUPS) { set_error("ttb_ar_step: %d prompt groups (0..%d)", a.groups, AS_MAX_GROUPS); return -1; }
  // prompt groups: rows [group_begin[g], group_begin[g + 1]) share the prefix group_prefix_kv[g] of group_P[g] positions
  pl.ngroups = a.groups > 0 ? a.groups : 1;
  p.ngroups = pl.ngroups;
  if (a.groups > 0) {
    if (!a.group_begin || !a.group_P || !a.group_prefix_kv) { set_error("ttb_ar_step: missing group arrays"); return -1; }
    if (a.group_begin[0] != 0 || a.group_begin[a.groups] != a.B) {
      set_error("ttb_ar_step: groups must cover rows [0, B=%d)", a.B); return -1;
    }
    for (int g = 0; g < a.groups; ++g) {
      if (a.group_begin[g + 1] <= a.group_begin[g]) { set_error("ttb_ar_step: group %d has no rows", g); return -1; }
      if (!a.group_prefix_kv[g]) { set_error("ttb_ar_step: group %d has no prefix", g); return -1; }
      pl.gtab[g].b0 = a.group_begin[g]; pl.gtab[g].P = a.group_P[g];
    }
  } else {
    pl.gtab[0].b0 = 0; pl.gtab[0].P = a.P;
  }
  pl.gtab[pl.ngroups].b0 = a.B;
  int maxP = 0;
  for (int g = 0; g < pl.ngroups; ++g) {
    const int P = pl.gtab[g].P;
    if (P <= 0 || P > AS_MAX_P) { set_error("ttb_ar_step: prompt length P=%d exceeds %d", P, AS_MAX_P); return -1; }
    if (P > maxP) maxP = P;
  }
  if (a.L <= 0 || a.V <= 0 || a.Nmax <= 0) { set_error("ttb_ar_step: bad shape"); return -1; }
  const int grid = as_num_sms();
  pl.grid = grid;
  p.B = a.B; p.D = a.D; p.H = a.H; p.L = a.L; p.V = a.V; p.Nmax = a.Nmax; p.pos_mode = a.pos_mode;
  const int Bpad = (a.B + 15) & ~15;
  p.nbt = (Bpad + 127) / 128;
  p.TB = (((Bpad + p.nbt - 1) / p.nbt) + 15) & ~15;
  p.stage_bytes = AS_W_TILE_BYTES + p.TB * 128;
  p.nst = AS_DATA_BYTES / p.stage_bytes;
  if (p.nst > AS_MAX_STAGES) p.nst = AS_MAX_STAGES;
  // most K splits: GEMMs with a final (bf16 / logit) output, and the two whose partials the next LayerNorm sums
  const int cap_f = 8;
  const int cap_p = p.nbt > 1 ? 4 : 8;
  plan_gemm(p.g[G_QKV], 3 * a.D, a.D, p.nbt, grid, cap_f);
  plan_gemm(p.g[G_PROJ], a.D, a.D, p.nbt, grid, cap_p);
  plan_gemm(p.g[G_FC], 4 * a.D, a.D, p.nbt, grid, cap_f);
  plan_gemm(p.g[G_PROJ2], a.D, 4 * a.D, p.nbt, grid, cap_p);
  plan_gemm(p.g[G_HEAD], a.V, a.D, p.nbt, grid, cap_f);
  long long pf = 0;
  for (int i = 0; i < 5; ++i) {
    const long long need = (long long)p.g[i].nsplit * a.B * p.g[i].ldp;
    if (need > pf) pf = need;
    if (p.g[i].n_rt * p.nbt > AS_MAX_TILES) { set_error("ttb_ar_step: too many tiles"); return -1; }
  }
  pl.part_floats = pf;
  // attention decomposition (compact attention: AS_COMPACT_CTAS CTAs per SM, see ar_attn_compact_kernel): units =
  // (group, head, chunk of the group's rows); the CTAs per head are shared out over the groups in proportion to their rows
  const int ncph = grid * (a.attn_compact ? AS_COMPACT_CTAS : 1) / a.H;
  int max_items = 1;
  p.units = 0;
  for (int g = 0; g < pl.ngroups; ++g) {
    AsGroup& gr = pl.gtab[g];
    const int gB = pl.gtab[g + 1].b0 - gr.b0;
    gr.ncph = (int)((long long)ncph * gB / a.B);
    if (gr.ncph < 1) gr.ncph = 1;
    if (gr.ncph > gB) gr.ncph = gB;
    gr.u0 = p.units;
    p.units += a.H * gr.ncph;
    const int items = (gB + gr.ncph - 1) / gr.ncph;
    if (items > max_items) max_items = items;
  }
  pl.gtab[pl.ngroups].u0 = p.units;
  p.P0 = pl.gtab[0].P; p.ncph0 = pl.gtab[0].ncph;
  const int wcap = a.attn_compact ? AS_COMPACT_WARPS : AS_WARPS;
  const int rounds = (max_items + wcap - 1) / wcap;
  p.ipr = (max_items + rounds - 1) / rounds;
  int team = 1;
  while (team * 2 * p.ipr <= wcap) team *= 2;
  // test hook: TTB_AR_STEP_TEAM caps the warps per stream, so that runs at different batch sizes merge the same way
  // (test_two_chains_match_one_chain compares them bit for bit)
  const int tcap = env_int("TTB_AR_STEP_TEAM", 0);
  if (tcap > 0 && tcap < team) team = tcap;
  p.team = team;
  // the rings of the active warps + the longest prompt prefix of one head share the data region
  const int nact = p.ipr * p.team;
  const long long attn_bytes = (long long)nact * AS_RING_NS * AS_CHUNK_BYTES + (long long)((maxP + 15) & ~15) * AS_POS_BYTES;
  if (attn_bytes > AS_DATA_BYTES) {
    set_error("ttb_ar_step: ring %d x %d positions x %d warps + prompt %d do not fit shared memory", AS_RING_NS, AS_CHUNK_POS,
              nact, maxP);
    return -1;
  }
  p.attn_data_bytes = a.attn_compact ? (int)((attn_bytes + 1023) & ~1023LL) : 0;
  p.layer_begin = 0; p.layer_end = a.L; p.phase_mask = 0x1ff;
  if (a.debug_layer_end > 0) { p.layer_begin = a.debug_layer_begin; p.layer_end = a.debug_layer_end; }
  if (a.debug_phase_mask) p.phase_mask = a.debug_phase_mask;
  return 0;
}

constexpr int AS_EXTRA_MAPS = 6;      // activations a, o, h, hn; candidate KV cache; prompt-prefix KV cache of group 0
// device tables: tensor maps (weights, extra maps, the prefixes of groups 1..), layer table, group table
static int num_maps(int L, int ngroups) { return 4 * L + 1 + AS_EXTRA_MAPS + (ngroups - 1); }
static size_t group_table_offset(int L, int ngroups) {
  return (size_t)num_maps(L, ngroups) * sizeof(CUtensorMap) + (size_t)L * sizeof(AsLayer);
}
static long long table_bytes(int L, int ngroups) {
  return (long long)group_table_offset(L, ngroups) + (long long)(ngroups + 1) * sizeof(AsGroup) + 256;
}

}  // namespace ttb
using namespace ttb;

extern "C" int ttb_ar_step_workspace(const TtbArStepArgs* a, long long* part_floats, long long* table_bytes_out,
                                     long long* sync_bytes) {
  AsPlan pl;
  if (make_plan(*a, pl)) return -1;
  if (part_floats) *part_floats = pl.part_floats;
  if (table_bytes_out) *table_bytes_out = table_bytes(a->L, pl.ngroups);
  if (sync_bytes) *sync_bytes = AS_SYNC_BAR_BYTES + AS_MAX_TILES * 4;
  return 0;
}

// Builds the device tables (tensor maps + per-layer pointer table) in a->tables. Synchronous; call once per
// (weights, workspace, batch) before capturing / launching ttb_ar_decode_step.
extern "C" int ttb_ar_step_setup(const TtbArStepArgs* ap, void* stream) {
  const TtbArStepArgs& a = *ap;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  AsPlan pl;
  if (make_plan(a, pl)) return -1;
  if (!a.layers || !a.tables || !a.sync) { set_error("ttb_ar_step_setup: missing tables"); return -1; }
  const int nmaps = num_maps(a.L, pl.ngroups);
  std::vector<unsigned char> host((size_t)table_bytes(a.L, pl.ngroups), 0);
  CUtensorMap* maps = reinterpret_cast<CUtensorMap*>(host.data());
  AsLayer* lay = reinterpret_cast<AsLayer*>(host.data() + (size_t)nmaps * sizeof(CUtensorMap));
  memcpy(host.data() + group_table_offset(a.L, pl.ngroups), pl.gtab, (size_t)(pl.ngroups + 1) * sizeof(AsGroup));
  const uint64_t D = a.D;
  for (int l = 0; l < a.L; ++l) {
    const TtbArStepLayer& s = a.layers[l];
    if (get_tensor_map_bf16(&maps[4 * l + G_QKV], s.wqkv, D, 3 * D, 1, D, 3 * D * D, 64, 128)) return -1;
    if (get_tensor_map_bf16(&maps[4 * l + G_PROJ], s.wproj, D, D, 1, D, D * D, 64, 128)) return -1;
    if (get_tensor_map_bf16(&maps[4 * l + G_FC], s.wfc, D, 4 * D, 1, D, 4 * D * D, 64, 128)) return -1;
    if (get_tensor_map_bf16(&maps[4 * l + G_PROJ2], s.wproj2, 4 * D, D, 1, 4 * D, 4 * D * D, 64, 128)) return -1;
    lay[l].ln1_g = s.ln1_g; lay[l].ln1_b = s.ln1_b; lay[l].bqkv = s.bqkv; lay[l].bproj = s.bproj;
    lay[l].ln2_g = s.ln2_g; lay[l].ln2_b = s.ln2_b; lay[l].bfc = s.bfc; lay[l].bproj2 = s.bproj2;
  }
  if (get_tensor_map_bf16(&maps[4 * a.L], a.w_head, D, (uint64_t)a.V, 1, D, (uint64_t)a.V * D, 64, 128)) return -1;
  const uint64_t Bq = a.B;
  const uint32_t TB = (uint32_t)pl.p.TB;
  CUtensorMap* am = maps + 4 * a.L + 1;
  if (get_tensor_map_bf16(&am[0], a.a, D, Bq, 1, D, Bq * D, 64, TB)) return -1;
  if (get_tensor_map_bf16(&am[1], a.o, D, Bq, 1, D, Bq * D, 64, TB)) return -1;
  if (get_tensor_map_bf16(&am[2], a.h, 4 * D, Bq, 1, 4 * D, Bq * 4 * D, 64, TB)) return -1;
  if (get_tensor_map_bf16(&am[3], a.hn, D, Bq, 1, D, Bq * D, 64, TB)) return -1;
  {
    // KV caches as 4-D tensors [item][position][K|V][64]: one box = 16 positions of K (or V) of one (layer, cand, head)
    const uint32_t box[4] = {64, 1, 16, 1};
    const uint64_t cd[4] = {64, 2, (uint64_t)a.Nmax, (uint64_t)a.L * a.B * a.H};
    const uint64_t cs[3] = {128, 256, (uint64_t)a.Nmax * 256};
    if (make_tensor_map_bf16_nd(&am[4], a.cand_kv, 4, cd, cs, box)) return -1;
    // prompt prefix of group g, [L][H][P_g][2][64]: maps[4 L + 6 + g]
    for (int g = 0; g < pl.ngroups; ++g) {
      const uint64_t P = (uint64_t)pl.gtab[g].P;
      const uint64_t pd[4] = {64, 2, P, (uint64_t)a.L * a.H};
      const uint64_t ps[3] = {128, 256, P * 256};
      const void* pkv = a.groups > 0 ? a.group_prefix_kv[g] : a.prefix_kv;
      if (make_tensor_map_bf16_nd(&am[5 + g], pkv, 4, pd, ps, box)) return -1;
    }
  }
  cudaError_t e = cudaMemcpyAsync(a.tables, host.data(), host.size(), cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(a.sync, 0, AS_SYNC_BAR_BYTES + AS_MAX_TILES * 4, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return check_cuda(e, "ttb_ar_step_setup");
  static bool attr_set = false;
  if (!attr_set) {
    e = cudaFuncSetAttribute(ar_step_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, AS_SMEM_TOTAL);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(ar_step_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, AS_SMEM_TOTAL);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(ar_attn_only_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, AS_SMEM_TOTAL);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(ar_attn_only_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, AS_SMEM_TOTAL);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(ar_attn_compact_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, AS_SMEM_TOTAL);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(ar_attn_compact_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, AS_SMEM_TOTAL);
    if (e != cudaSuccess) return check_cuda(e, "cudaFuncSetAttribute(ar_step_kernel)");
    attr_set = true;
  }
  return 0;
}

extern "C" int ttb_ar_decode_step(const TtbArStepArgs* ap, void* stream) {
  const TtbArStepArgs& a = *ap;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  AsPlan pl;
  if (make_plan(a, pl)) return -1;
  AsParams& p = pl.p;
  const int nmaps = num_maps(a.L, pl.ngroups);
  p.maps = reinterpret_cast<const CUtensorMap*>(a.tables);
  p.layers = reinterpret_cast<const AsLayer*>(reinterpret_cast<const unsigned char*>(a.tables) + (size_t)nmaps * sizeof(CUtensorMap));
  p.gtab = reinterpret_cast<const AsGroup*>(reinterpret_cast<const unsigned char*>(a.tables) + group_table_offset(a.L, pl.ngroups));
  p.lnf_g = a.lnf_g; p.lnf_b = a.lnf_b; p.fn_g = a.fn_g; p.fn_b = a.fn_b; p.b_head = a.b_head;
  p.mel_emb = a.mel_emb; p.mel_pos = a.mel_pos; p.codes = a.codes; p.ld_codes = a.ld_codes; p.state = a.state;
  p.x = a.x;
  p.a = reinterpret_cast<__nv_bfloat16*>(a.a); p.qkv = reinterpret_cast<__nv_bfloat16*>(a.qkv);
  p.o = reinterpret_cast<__nv_bfloat16*>(a.o); p.h = reinterpret_cast<__nv_bfloat16*>(a.h);
  p.hn = reinterpret_cast<__nv_bfloat16*>(a.hn);
  p.part = a.part; p.logits = a.logits;
  p.prefix_kv = reinterpret_cast<const __nv_bfloat16*>(a.prefix_kv);
  p.cand_kv = reinterpret_cast<__nv_bfloat16*>(a.cand_kv);
  p.row_start = a.row_start;
  p.bar = reinterpret_cast<unsigned long long*>(a.sync);
  p.tickets = reinterpret_cast<unsigned int*>(reinterpret_cast<unsigned char*>(a.sync) + AS_SYNC_BAR_BYTES);
  if (p.phase_mask == PH_ATTN && p.layer_end == p.layer_begin + 1) {
    const int units = p.units;
    if (a.attn_compact) {
      const int cgrid = pl.grid * AS_COMPACT_CTAS;
      const dim3 grid(units < cgrid ? units : cgrid), block(AS_COMPACT_WARPS * 32);
      const size_t smem = (size_t)(p.attn_data_bytes + AS_CTRL_COMPACT_BYTES + 1024);
      const cudaError_t lc = a.row_start ? launch_pdl(ar_attn_compact_kernel<true>, grid, block, smem, st, p)
                                         : launch_pdl(ar_attn_compact_kernel<false>, grid, block, smem, st, p);
      if (lc != cudaSuccess) return check_cuda(lc, "ar_attn_compact_kernel launch");
      TTB_CHECK_LAUNCH("ar_attn_compact_kernel");
      return 0;
    }
    const dim3 grid(units < pl.grid ? units : pl.grid), block(AS_THREADS);
    const cudaError_t la = a.row_start ? launch_pdl(ar_attn_only_kernel<true>, grid, block, (size_t)AS_SMEM_TOTAL, st, p)
                                       : launch_pdl(ar_attn_only_kernel<false>, grid, block, (size_t)AS_SMEM_TOTAL, st, p);
    if (la != cudaSuccess) return check_cuda(la, "ar_attn_only_kernel launch");
    TTB_CHECK_LAUNCH("ar_attn_only_kernel");
    return 0;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(pl.grid);
  cfg.blockDim = dim3(AS_THREADS);
  cfg.dynamicSmemBytes = AS_SMEM_TOTAL;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeCooperative;
  at[0].val.cooperative = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  const cudaError_t le = a.row_start ? cudaLaunchKernelEx(&cfg, ar_step_kernel<true>, p)
                                     : cudaLaunchKernelEx(&cfg, ar_step_kernel<false>, p);
  if (le != cudaSuccess) return check_cuda(le, "ar_step_kernel launch");
  TTB_CHECK_LAUNCH("ar_step_kernel");
  return 0;
}

extern "C" int ttb_ar_step_store_prefix_cap(const void* qkv, int P, int cap, int H, void* prefix_kv, void* stream) {
  if (P <= 0 || cap < P) { set_error("ttb_ar_step_store_prefix_cap: P=%d, cap=%d (need 0 < P <= cap)", P, cap); return -1; }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long n = (long long)P * H * 64;
  ar_step_store_prefix_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(qkv), P, cap,
                                                                          H, reinterpret_cast<__nv_bfloat16*>(prefix_kv));
  TTB_CHECK_LAUNCH("ar_step_store_prefix_kernel");
  return 0;
}

extern "C" int ttb_ar_step_store_prefix(const void* qkv, int P, int H, void* prefix_kv, void* stream) {
  return ttb_ar_step_store_prefix_cap(qkv, P, P, H, prefix_kv, stream);
}

extern "C" int ttb_ar_step_set_group_len(const TtbArStepArgs* ap, int group, int P, void* stream) {
  const TtbArStepArgs& a = *ap;
  AsPlan pl;
  if (make_plan(a, pl)) return -1;
  if (!a.tables || group < 0 || group >= pl.ngroups) {
    set_error("ttb_ar_step_set_group_len: group %d of %d (or no tables)", group, pl.ngroups);
    return -1;
  }
  if (P <= 0 || P > pl.gtab[group].P) {
    set_error("ttb_ar_step_set_group_len: P=%d outside (0, %d], the prefix capacity of group %d", P, pl.gtab[group].P, group);
    return -1;
  }
  AsGroup* gtab = reinterpret_cast<AsGroup*>(reinterpret_cast<unsigned char*>(a.tables) + group_table_offset(a.L, pl.ngroups));
  ar_step_set_group_len_kernel<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(gtab, group, P);
  TTB_CHECK_LAUNCH("ar_step_set_group_len_kernel");
  return 0;
}
