// Cluster / TMA-multicast variant of the wgmma GEMM (included by gemm.cu).
//
// With one CTA per 128xBN tile every CTA pulls its own copy of the 128x64 activation tile per k-block, and the L2->SM
// fabric saturates before the tensor pipe does (decode GEMMs with BN=32 move 16 KB of A for 4 KB of weights per k-block).
// Here CL CTAs that are neighbours along N (same m-tile) form a thread-block cluster: each loads 1/CL of the A tile
// and MULTICASTS it into the shared memory of all CL CTAs (cp.async.bulk.tensor ... .multicast::cluster); the weight
// tile stays private. Per k-block a CTA reads 16/CL KB + B instead of 16 KB + B.
//
// Synchronisation: every CTA arms its own full barrier with the whole stage's bytes (its B tile + CL multicast slices of
// A land in ITS smem and complete_tx on ITS barrier). A stage may only be overwritten when ALL CTAs of the cluster have
// consumed it, so each consumer warpgroup arrives on the empty barrier of every CTA in the cluster once its wgmma group
// has retired, and empty barriers are initialised with count 2 * CL.
#pragma once

namespace ttb {

TTB_DEVINL uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
TTB_DEVINL void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
TTB_DEVINL void tma_load_3d_mc(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%4, %5, %6}], [%2], %3;"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "h"(mask), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// arrive on the copy of `bar` in CTA `cta` of this cluster
TTB_DEVINL void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
  asm volatile(
      "{\n\t.reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n\t}\n" ::"r"(smem_u32(bar)), "r"(cta)
      : "memory");
}

template <int BN, int STAGES, int CL>
__global__ void __launch_bounds__(GEMM_THREADS)
gemm_bf16_tc_mc_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, int M, int N,
                       int K, int taps, int pad, int a_batch_mul, int kb_per_split, GemmEpilogue ep) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  using L = GemmSmem<BN, STAGES>;
  constexpr int SLICE_ROWS = BM / CL;
  constexpr int SLICE_BYTES = SLICE_ROWS * BK * 2;
  constexpr uint16_t MASK = (uint16_t)((1u << CL) - 1);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int n0 = blockIdx.x * BN;
  const int m0 = blockIdx.y * BM;
  const int bz = blockIdx.z;
  const uint32_t crank = cluster_ctarank();
  const int kblocks_per_tap = K / BK;
  const int kb_total = kblocks_per_tap * taps;
  const int kb_begin = kb_per_split > 0 ? bz * kb_per_split : 0;
  const int num_kb = kb_per_split > 0 ? min(kb_per_split, kb_total - kb_begin) : kb_total;

  if (warp == PRODUCER_WARP && lane == 0) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_b);
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2 * CL); }
    fence_barrier_init();
  }
  __syncthreads();
  cluster_sync_all();            // peers' barriers are initialised before anyone multicasts into them

  if (warp == PRODUCER_WARP) {
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int kbi = 0; kbi < num_kb; ++kbi) {
        mbar_wait(&empty_bar[stage], phase ^ 1);      // every CTA of the cluster has released this stage
        const int kb = kb_begin + kbi;
        const int tap = kb / kblocks_per_tap;
        const int kk = (kb - tap * kblocks_per_tap) * BK;
        uint8_t* sa = smem + stage * L::STAGE_BYTES;
        uint8_t* sb = sa + L::A_BYTES;
        mbar_arrive_expect_tx(&full_bar[stage], L::STAGE_BYTES);
        // my 1/CL slice of the shared A tile -> same offset in every CTA of the cluster
        tma_load_3d_mc(sa + crank * SLICE_BYTES, &map_a, &full_bar[stage], kk, m0 + (int)crank * SLICE_ROWS + tap - pad,
                       bz * a_batch_mul, MASK);
        tma_load_3d(sb, &map_b, &full_bar[stage], tap * K + kk, n0, 0);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
    __syncwarp();
  } else {
    const int wg = warp >> 2;
    const int rb = warp >> 1;
    float acc[BN / 2];
    int stage = 0; uint32_t phase = 0;
    gemm_consumer_mainloop<BN, STAGES>(acc, smem, L::STAGE_BYTES, L::A_BYTES, full_bar, empty_bar, num_kb, stage, phase, wg,
                                       (threadIdx.x & 127) == 0, [](uint64_t* b) {
                                         for (uint32_t c = 0; c < (uint32_t)CL; ++c) mbar_arrive_cluster(b, c);   // release the stage in every CTA
                                       });
    // every wgmma of both warpgroups has retired and every multicast slice of this CTA's stages has landed: the pipeline
    // stages are idle and take the staged accumulator tile
    named_barrier(1, GEMM_CONSUMERS);
    gemm_stage_accumulator<BN>(acc, smem_u32(smem), warp, lane);
    named_barrier(1, GEMM_CONSUMERS);
    gemm_epilogue_dispatch<BN>(smem_u32(smem) + (uint32_t)(rb * 32 * (BN + 8)) * 4, n0, N, m0 + rb * 32, M, lane, (long long)bz,
                               ep, warp & 1, 2);
  }
  __syncthreads();
  cluster_sync_all();            // nobody exits while a peer may still arrive on its barriers
}

template <int BN, int STAGES, int CL>
static int launch_mc(const TtbGemmArgs& g, const GemmEpilogue& ep, cudaStream_t st) {
  CUtensorMap ma, mb;
  const bool bcast = (g.batch == 1) || (g.a_bstride == 0);
  const uint64_t a_d2 = bcast ? 1 : (uint64_t)g.batch;
  const uint64_t a_s2 = bcast ? (uint64_t)g.rows * g.lda : (uint64_t)g.a_bstride;
  if (get_tensor_map_bf16(&ma, g.A, (uint64_t)g.K, (uint64_t)g.rows, a_d2, (uint64_t)g.lda, a_s2, BK, BM / CL)) return -1;
  if (get_tensor_map_bf16(&mb, g.W, (uint64_t)g.K * g.taps, (uint64_t)g.N, 1, (uint64_t)g.K * g.taps,
                          (uint64_t)g.K * g.taps * g.N, BK, BN)) return -1;
  using L = GemmSmem<BN, STAGES>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gemm_bf16_tc_mc_kernel<BN, STAGES, CL>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL);
    if (e != cudaSuccess) return check_cuda(e, "cudaFuncSetAttribute(gemm mc)");
    attr_set = true;
  }
  int kb_per_split = 0, zdim = g.batch;
  if (g.splitk > 1) {
    const int kb_total = (g.K / BK) * g.taps;
    kb_per_split = (kb_total + g.splitk - 1) / g.splitk;
    zdim = (kb_total + kb_per_split - 1) / kb_per_split;
  }
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((g.N + BN - 1) / BN, (g.M + BM - 1) / BM, zdim);
  cfg.blockDim = dim3(GEMM_THREADS);
  cfg.dynamicSmemBytes = L::TOTAL;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CL; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  cudaError_t e = cudaLaunchKernelEx(&cfg, gemm_bf16_tc_mc_kernel<BN, STAGES, CL>, ma, mb, g.M, g.N, g.K, g.taps, g.pad,
                                     (bcast || g.splitk > 1) ? 0 : 1, kb_per_split, ep);
  if (e != cudaSuccess) return check_cuda(e, "cudaLaunchKernelEx(gemm mc)");
  return 0;
}

}  // namespace ttb
