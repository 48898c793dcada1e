// Persistent, warp-specialised 128x256 wgmma GEMM (included by gemm.cu after GemmEpilogue / BM / BK are defined).
//
// 384 threads in three warpgroups:
//   * warpgroup 0 = TMA producer: one thread issues every load; the warpgroup gives registers back (setmaxnreg.dec 40);
//   * warpgroups 1, 2 = consumers (setmaxnreg.inc 232): each owns 64 rows of the 128x256 tile and issues one m64n256k16
//     per k16 step (128 fp32 accumulators per thread). The A slice is read from shared memory once per k16 step instead
//     of once per 64 columns, and a 128x256x64 k-block carries 85 instead of 64 FLOP per operand byte.
// One CTA per SM walks the output tiles in the order of the persistent kernel (m fastest within an n panel, then batch),
// so the CTAs running at the same time share weight panels in L2. While the consumers drain tile i the producer fills the
// stages they freed with the k-blocks of tile i + 1. The pipeline stages are therefore not free for the epilogue: each
// warpgroup drains its 64 rows through two staging slices of its own, 2 x 32 columns per round (the two warps of a
// 32-row block finish one slice each), and every 32x32 block goes through the epilogue chunk routines of
// gemm_epilogue.cuh, so each output element and each GroupNorm partial is computed by the same code, in the same order,
// as in the one-tile kernel. The slices have no padding (pitch 32) so that two per warpgroup fit next to 4 stages.
// Split-K and clusters are not supported (those calls keep their kernels).
#pragma once

namespace ttb {

constexpr int WS_BN = 256;
constexpr int WS_STAGES = 4;
constexpr int WS_THREADS = 384;
constexpr int WS_SLICE = 32;          // accumulator columns per staging slice; each warpgroup stages two per round

struct GemmWsSmem {
  static constexpr int A_BYTES = BM * BK * 2;                 // 16 KB
  static constexpr int B_BYTES = WS_BN * BK * 2;              // 32 KB
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STG_PITCH = WS_SLICE;                  // floats
  static constexpr int SLICE_BYTES = 64 * STG_PITCH * 4;      // one warpgroup's 64 rows of one slice
  static constexpr int STG_OFF = WS_STAGES * STAGE_BYTES;     // staging slices [warpgroup][2][64][STG_PITCH] fp32
  static constexpr int BAR_OFF = STG_OFF + 4 * SLICE_BYTES;
  static constexpr int TOTAL = BAR_OFF + 2 * WS_STAGES * 8 + 1024;   // + alignment slack
  static_assert(TOTAL <= 227 * 1024, "warp-specialised GEMM shared memory");
};

__global__ void __launch_bounds__(WS_THREADS, 1)
gemm_bf16_ws_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, int M, int N,
                    int K, int taps, int pad, int a_batch_mul, int m_tiles, int n_tiles, int z_tiles, GemmEpilogue ep) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  using L = GemmWsSmem;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
  uint64_t* empty_bar = full_bar + WS_STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int kblocks_per_tap = K / BK;
  const int num_kb = kblocks_per_tap * taps;
  const int total_tiles = m_tiles * n_tiles * z_tiles;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_b);
    for (int s = 0; s < WS_STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
    fence_barrier_init();
  }
  __syncthreads();
  // TtbGemmArgs.w_static (see the one-tile kernel): the weight halves of the first tile's first stages are requested
  // before griddepcontrol.wait.
  int pre = 0;
  if (ep.wpre && threadIdx.x == 0) {
    const int n0 = ((blockIdx.x / m_tiles) % n_tiles) * WS_BN;
    pre = num_kb < WS_STAGES ? num_kb : WS_STAGES;
    for (int kb = 0; kb < pre; ++kb) {
      const int tap = kb / kblocks_per_tap;
      const int kk = (kb - tap * kblocks_per_tap) * BK;
      mbar_arrive_expect_tx(&full_bar[kb], L::STAGE_BYTES);
      tma_load_3d(smem + kb * L::STAGE_BYTES + L::A_BYTES, &map_b, &full_bar[kb], tap * K + kk, n0, 0);
    }
  }
  pdl_wait();                    // activations, residual and outputs belong to earlier kernels until here

  if (warp < 4) {
    // ===== TMA producer =====
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int mt = tile % m_tiles, rest = tile / m_tiles;
        const int nt = rest % n_tiles, bz = rest / n_tiles;
        const int m0 = mt * BM, n0 = nt * WS_BN;
        const int npre = tile == (int)blockIdx.x ? pre : 0;   // stages whose weight half is already on its way
        for (int kb = 0; kb < num_kb; ++kb) {
          const int tap = kb / kblocks_per_tap;
          const int kk = (kb - tap * kblocks_per_tap) * BK;
          uint8_t* sa = smem + stage * L::STAGE_BYTES;
          if (kb >= npre) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            mbar_arrive_expect_tx(&full_bar[stage], L::STAGE_BYTES);
            tma_load_3d(sa + L::A_BYTES, &map_b, &full_bar[stage], tap * K + kk, n0, 0);
          }
          tma_load_3d(sa, &map_a, &full_bar[stage], kk, m0 + tap * ep.tap_dil - pad, bz * a_batch_mul);
          if (++stage == WS_STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    __syncwarp();
    pdl_launch_dependents();     // tail trigger: every load of this CTA is issued
  } else {
    // ===== consumers: warpgroup wg owns rows [64 wg, 64 wg + 64) of every tile =====
    setmaxnreg_inc<232>();
    const int cw = warp - 4;                           // consumer warp 0..7 (accumulator rows 16 cw ..)
    const int wg = cw >> 2;
    const int rb = cw >> 1;                            // 32-row block this warp finishes (one slice per round)
    const bool leader = (threadIdx.x & 127) == 0;
    const uint32_t stg = smem_u32(smem + L::STG_OFF) + (uint32_t)(wg * 2 * L::SLICE_BYTES);
    const uint32_t blk = stg + (uint32_t)((cw & 1) * L::SLICE_BYTES + (rb & 1) * 32 * L::STG_PITCH * 4);
    int stage = 0; uint32_t phase = 0;
    float acc[WS_BN / 2];
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int mt = tile % m_tiles, rest = tile / m_tiles;
      const int nt = rest % n_tiles, bz = rest / n_tiles;
      const int m0 = mt * BM, n0 = nt * WS_BN;
      if (ep.residual && !(cw & 1)) {
        // pull the tile's residual rows into L2 ahead of the epilogue
        const int m = m0 + rb * 32 + lane;
        if (m < M) {
          const float* p = ep.residual + (long long)bz * ep.res_bstride + (long long)m * ep.ldr + n0;
#pragma unroll
          for (int c = 0; c < WS_BN; c += 32)
            if (n0 + c < N) asm volatile("prefetch.global.L2 [%0];" ::"l"(p + c));
        }
      }
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * L::STAGE_BYTES);
        gemm_mma_kblock_n256(acc, sa + wg * (64 * BK * 2), sa + L::A_BYTES, kb == 0);
        wgmma_wait<1>();
        if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == WS_STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if (leader) mbar_arrive(&empty_bar[prev]);
      if (tile + (int)gridDim.x >= total_tiles) pdl_launch_dependents();   // this CTA's last accumulator is complete
      // drain: 64 columns per round, slice 2 r + h in staging slice h, finished by the warps with (cw & 1) == h
#pragma unroll 1
      for (int r = 0; r < WS_BN / (2 * WS_SLICE); ++r) {
        if (n0 + r * 2 * WS_SLICE >= N) break;         // uniform over the CTA
        named_barrier(1 + wg, 128);                    // the previous round's readers are done
#pragma unroll
        for (int j = 0; j < WS_BN / (2 * WS_SLICE); ++j) {   // static register indices: acc stays in registers
          if (j == r) {
            gemm_stage_accumulator<WS_SLICE, L::STG_PITCH>(acc + 2 * j * (WS_SLICE / 2), stg, cw & 3, lane);
            gemm_stage_accumulator<WS_SLICE, L::STG_PITCH>(acc + (2 * j + 1) * (WS_SLICE / 2), stg + L::SLICE_BYTES, cw & 3, lane);
          }
        }
        named_barrier(1 + wg, 128);
        const int nb = n0 + (2 * r + (cw & 1)) * WS_SLICE;
        if (nb < N) {
          // The empty asm makes these values opaque per round. Otherwise the compiler computes the epilogue's row
          // addresses once per tile, and they spill: 128 accumulator registers are live across the whole drain.
          int mb = m0 + rb * 32, ln = lane, b = bz;
          uint32_t bk = blk;
          asm volatile("" : "+r"(mb), "+r"(ln), "+r"(b), "+r"(bk));
          gemm_epilogue_dispatch<WS_SLICE, L::STG_PITCH>(bk, nb, N, mb, M, ln, (long long)b, ep, 0, 1);
        }
      }
    }
  }
}

}  // namespace ttb
