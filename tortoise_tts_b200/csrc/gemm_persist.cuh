// Persistent variant of the wgmma GEMM (included by gemm.cu after GemmEpilogue / BM / BK are defined).
//
// One CTA per SM loops over output tiles (tile id -> m fastest, then n, then batch/split), so that
//   * the TMA producer runs ahead into the next tile's k-blocks while the consumers finish the epilogue of this one,
//   * barrier init / descriptor prefetch are paid once per CTA instead of once per tile.
// Roles: warps 0..7 = two consumer warpgroups (wgmma, then the epilogue of their own 64 rows from a dedicated staging
// tile), warp 8 = TMA producer.
#pragma once

namespace ttb {

template <int BN, int PSTAGES>
struct GemmPSmem {
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int ACC_OFF = PSTAGES * STAGE_BYTES;                      // staged accumulator tile [128][BN + 8] fp32
  static constexpr int BAR_OFF = ACC_OFF + BM * (BN + 8) * 4;
  static constexpr int TOTAL = BAR_OFF + 2 * PSTAGES * 8 + 16 + 1024;
  static_assert(TOTAL <= 227 * 1024, "persistent GEMM shared memory");
};

template <int BN, int PSTAGES>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_tc_persistent_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                               int M, int N, int K, int taps, int pad, int a_batch_mul, int kb_per_split, int m_tiles,
                               int n_tiles, int z_tiles, GemmEpilogue ep) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  using L = GemmPSmem<BN, PSTAGES>;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
  uint64_t* empty_bar = full_bar + PSTAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int kblocks_per_tap = K / BK;
  const int kb_total = kblocks_per_tap * taps;
  const int total_tiles = m_tiles * n_tiles * z_tiles;

  if (warp == PRODUCER_WARP && lane == 0) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_b);
    for (int s = 0; s < PSTAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();

  if (warp == PRODUCER_WARP) {
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int mt = tile % m_tiles, rest = tile / m_tiles;
        const int nt = rest % n_tiles, bz = rest / n_tiles;
        const int m0 = mt * BM, n0 = nt * BN;
        const int kb_begin = kb_per_split > 0 ? bz * kb_per_split : 0;
        const int num_kb = kb_per_split > 0 ? min(kb_per_split, kb_total - kb_begin) : kb_total;
        for (int kbi = 0; kbi < num_kb; ++kbi) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          const int kb = kb_begin + kbi;
          const int tap = kb / kblocks_per_tap;
          const int kk = (kb - tap * kblocks_per_tap) * BK;
          uint8_t* sa = smem + stage * L::STAGE_BYTES;
          uint8_t* sb = sa + L::A_BYTES;
          mbar_arrive_expect_tx(&full_bar[stage], L::STAGE_BYTES);
          tma_load_3d(sa, &map_a, &full_bar[stage], kk, m0 + tap * ep.tap_dil - pad, bz * a_batch_mul);
          tma_load_3d(sb, &map_b, &full_bar[stage], tap * K + kk, n0, 0);
          if (++stage == PSTAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    __syncwarp();
  } else {
    const int wg = warp >> 2;
    const int rb = warp >> 1;
    const uint32_t acc_tile = smem_u32(smem + L::ACC_OFF);
    int stage = 0; uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int mt = tile % m_tiles, rest = tile / m_tiles;
      const int nt = rest % n_tiles, bz = rest / n_tiles;
      const int kb_begin = kb_per_split > 0 ? bz * kb_per_split : 0;
      const int num_kb = kb_per_split > 0 ? min(kb_per_split, kb_total - kb_begin) : kb_total;
      float acc[BN / 2];
      gemm_consumer_mainloop<BN, PSTAGES>(acc, smem, L::STAGE_BYTES, L::A_BYTES, full_bar, empty_bar, num_kb, stage, phase, wg,
                                          (threadIdx.x & 127) == 0, [](uint64_t* b) { mbar_arrive(b); });
      // rows [64 wg, 64 wg + 64) of the staging tile are written and read by warpgroup wg only
      named_barrier(1 + wg, 128);                      // the previous tile's readers are done
      gemm_stage_accumulator<BN>(acc, acc_tile, warp, lane);
      named_barrier(1 + wg, 128);
      gemm_epilogue_dispatch<BN>(acc_tile + (uint32_t)(rb * 32 * (BN + 8)) * 4, nt * BN, N, mt * BM + rb * 32, M, lane,
                                 (long long)bz, ep, warp & 1, 2);
    }
  }
  pdl_launch_dependents();      // tail trigger (see gemm.cu)
}

}  // namespace ttb
