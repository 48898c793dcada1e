// wgmma GEMM / conv-as-GEMM for sm_90a.
//
//   D[b, m, n] = epilogue( sum_{tap, k} A[b, m + tap*1 - pad, k] * W[n, tap*K + k] )
//
// A: bf16 activations, token-major [batch, rows, K] (K contiguous), streamed by TMA (3-D map; out-of-range
//    rows are zero-filled by the TMA unit, which is exactly Conv1d zero padding).
// W: bf16 weights [N, taps*K] (K-major), streamed by TMA.
// Accumulator: fp32 in the registers of two consumer warpgroups (64 rows x BN columns each), written by
// wgmma.mma_async (m64nNk16, both operands from shared memory).
// Warp roles (288 threads): warps 0..7 = the two consumer warpgroups (main loop, then the epilogue: accumulator staged
// through shared memory -> bias / activation / residual -> global), warp 8 = TMA producer.
//
// Replaces, behind the C-ABI, every dense contraction of the reference hot path that PyTorch dispatches to
// cuBLAS / cuDNN: HF Conv1D addmm (GPT-2 c_attn/c_proj/c_fc, via autoregressive.py:150-163), nn.Linear
// (mel_head, CLVP to_q/k/v/out/FF xtransformers.py:519-521,440-474), nn.Conv1d k=1/k=3 of DiffusionTts
// (diffusion_decoder.py:83-103, arch_util.py:107-111) and the UnivNet kernel-predictor convs (vocoder.py:40-64).
#include "common.cuh"
#include "ttb_internal.h"

#include <map>
#include <mutex>
#include <string>
#include <vector>
#include <cstring>

namespace ttb {

// ------------------------------------------------------------------ tensor-map cache (host)
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, []() {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  });
  return fn;
}

struct MapKey {
  const void* ptr;
  uint64_t d0, d1, d2, s1, s2;
  uint32_t b0, b1;
  bool operator<(const MapKey& o) const { return memcmp(this, &o, sizeof(MapKey)) < 0; }
};

// bf16, up to 3 dims (dim0 contiguous), box = {b0, b1, 1}, SWIZZLE_128B (b0 * 2 bytes must be 128)
int get_tensor_map_bf16(CUtensorMap* out, const void* ptr, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t stride1_elems,
                        uint64_t stride2_elems, uint32_t b0, uint32_t b1) {
  static std::map<MapKey, CUtensorMap> cache;
  static std::mutex mu;
  MapKey key;
  memset(&key, 0, sizeof(key));
  key.ptr = ptr; key.d0 = d0; key.d1 = d1; key.d2 = d2; key.s1 = stride1_elems; key.s2 = stride2_elems;
  key.b0 = b0; key.b1 = b1;
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find(key);
  if (it != cache.end()) { *out = it->second; return 0; }
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return -1; }
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) || ((stride1_elems * 2) & 15) || ((stride2_elems * 2) & 15)) {
    set_error("tensor map: pointer/strides must be 16-byte aligned (ptr=%p s1=%llu s2=%llu)", ptr,
              (unsigned long long)stride1_elems, (unsigned long long)stride2_elems);
    return -1;
  }
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {stride1_elems * 2, stride2_elems * 2};
  cuuint32_t box[3] = {b0, b1, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUtensorMap m;
  CUresult r = enc(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d): dims=%llu,%llu,%llu strides=%llu,%llu box=%u,%u", (int)r,
              (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)d2,
              (unsigned long long)strides[0], (unsigned long long)strides[1], b0, b1);
    return -1;
  }
  cache[key] = m;
  *out = m;
  return 0;
}

// General form: bf16, rank <= 5, explicit byte strides of dims 1.. (dim 0 contiguous), SWIZZLE_128B (box[0] * 2 == 128).
int make_tensor_map_bf16_nd(CUtensorMap* out, const void* ptr, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                            const uint32_t* box) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return -1; }
  cuuint64_t d[5];
  cuuint64_t st[4];
  cuuint32_t b[5], es[5];
  for (int i = 0; i < rank; ++i) { d[i] = dims[i]; b[i] = box[i]; es[i] = 1; }
  for (int i = 0; i + 1 < rank; ++i) st[i] = strides_bytes[i];
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(ptr), d, st, b, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled (rank %d) failed (%d)", rank, (int)r); return -1; }
  return 0;
}

// ------------------------------------------------------------------ kernel
constexpr int BM = 128;
constexpr int BK = 64;
constexpr int GEMM_CONSUMERS = 256;      // two warpgroups: wgmma + epilogue
constexpr int PRODUCER_WARP = 8;          // TMA producer
constexpr int GEMM_THREADS = GEMM_CONSUMERS + 32;

struct GemmEpilogue {
  const float* bias;       // [N] or null
  const float* residual;   // fp32 [batch, M, ldr] or null (added after activation)
  float* out_f32;          // [batch, M, ldo] or null
  __nv_bfloat16* out_bf16; // [batch, M, ldob] or null
  long long res_bstride, outf_bstride, outb_bstride;
  int ldr, ldo, ldob;
  int act;                 // TTB_ACT_*
  float alpha;             // scales the accumulator before bias
  int tap_dil;             // row distance between conv taps (dilation); 1 = plain
  float2* gn_part;         // GroupNorm partials [batch][groups][TTB_GN_SPLITS] of the output, or null (TtbGemmArgs.gn_partials)
  int gn_groups;
  int wpre;                // TtbGemmArgs.w_static: W may be fetched before griddepcontrol.wait (one-tile kernel)
};

}  // namespace ttb
#include "gemm_epilogue.cuh"
namespace ttb {

template <int BN, int STAGES>
struct GemmSmem {
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int BAR_OFF = STAGES * STAGE_BYTES;
  static constexpr int TOTAL = BAR_OFF + (2 * STAGES + 1) * 8 + 16 + 1024;  // + alignment slack
  // once the main loop has retired, the pipeline stages hold the staged fp32 accumulator tile [128][BN + 8]
  static_assert(BM * (BN + 8) * 4 <= BAR_OFF, "accumulator tile must fit the idle pipeline stages");
  static_assert(TOTAL <= 227 * 1024, "GEMM shared memory");
};

// Main loop of the two consumer warpgroups over num_kb pipeline stages, starting at (stage, phase). One thread per
// warpgroup releases a stage once the wgmma group that read it has retired (one group stays in flight). RELEASE(bar)
// performs the arrive (plain, or on every CTA of a cluster).
template <int BN, int STAGES, typename Release>
TTB_DEVINL void gemm_consumer_mainloop(float* acc, uint8_t* smem, int stage_bytes, int a_bytes, uint64_t* full_bar,
                                       uint64_t* empty_bar, int num_kb, int& stage, uint32_t& phase, int wg, bool leader,
                                       Release release) {
  int prev = -1;
  for (int kb = 0; kb < num_kb; ++kb) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t sa = smem_u32(smem + stage * stage_bytes);
    gemm_mma_kblock<BN>(acc, sa + wg * (64 * BK * 2), sa + a_bytes, kb == 0);
    wgmma_wait<1>();
    if (prev >= 0 && leader) release(&empty_bar[prev]);
    prev = stage;
    if (++stage == STAGES) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
  if (prev >= 0 && leader) release(&empty_bar[prev]);
}

// SPLIT_PRODUCER (experiment, variant 5): the A tiles are issued by lane 0 and the B tiles by lane 1 of the producer warp:
// if the rate at which one CTA receives its operands is limited per issuing thread, two issuers double it.
template <int BN, int STAGES, bool SPLIT_PRODUCER = false>
__global__ void __launch_bounds__(GEMM_THREADS, BN <= 64 ? 2 : 1)
gemm_bf16_tc_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, int M, int N,
                    int K, int taps, int pad, int a_batch_mul, int kb_per_split, GemmEpilogue ep,
                    unsigned long long* trace) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  using L = GemmSmem<BN, STAGES>;
  // optional per-CTA phase timestamps (ttb_debug_gemm_trace): 8 x u64 per CTA, see tools/gemm_diag.py
  unsigned long long* tr = trace ? trace + 8ull * (blockIdx.x + gridDim.x * (blockIdx.y + (unsigned long long)gridDim.y * blockIdx.z)) : nullptr;
  if (tr && threadIdx.x == 0) { tr[0] = global_timer_ns(); tr[1] = sm_id(); }
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int n0 = blockIdx.x * BN;
  const int m0 = blockIdx.y * BM;
  const int bz = blockIdx.z;
  const int kblocks_per_tap = K / BK;
  // split-K: grid.z enumerates K ranges of kb_per_split k-blocks (batch == 1); each split writes a raw partial
  const int kb_total = kblocks_per_tap * taps;
  const int kb_begin = kb_per_split > 0 ? bz * kb_per_split : 0;
  const int num_kb = kb_per_split > 0 ? min(kb_per_split, kb_total - kb_begin) : kb_total;

  if (warp == PRODUCER_WARP && lane == 0) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_b);
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], SPLIT_PRODUCER ? 2 : 1); mbar_init(&empty_bar[s], 2); }
    fence_barrier_init();
  }
  __syncthreads();
  // W is a parameter (TtbGemmArgs.w_static): under programmatic dependent launch its tiles do not have to wait for the
  // kernels before this one. The first STAGES weight tiles go into the pipeline BEFORE griddepcontrol.wait; only the
  // activation tiles are requested after it. For the skinny decode GEMMs (a 64 KB slab per CTA in front of a short
  // main loop) the weights then stream while the previous kernel (LayerNorm, which triggers its dependents early) is
  // still running.
  int pre = 0;
  if constexpr (!SPLIT_PRODUCER) {
    if (ep.wpre && warp == PRODUCER_WARP && lane == 0) {
      pre = num_kb < STAGES ? num_kb : STAGES;
      for (int kbi = 0; kbi < pre; ++kbi) {
        const int kb = kb_begin + kbi;
        const int tap = kb / kblocks_per_tap;
        const int kk = (kb - tap * kblocks_per_tap) * BK;
        uint8_t* sb = smem + kbi * L::STAGE_BYTES + L::A_BYTES;
        mbar_arrive_expect_tx(&full_bar[kbi], L::STAGE_BYTES);
        tma_load_3d(sb, &map_b, &full_bar[kbi], tap * K + kk, n0, 0);
      }
    }
  }
  pdl_wait();                    // activations, residual and outputs belong to earlier kernels until here
  if (tr && threadIdx.x == 0) tr[2] = global_timer_ns();

  if (warp == PRODUCER_WARP) {
    // ===== TMA producer =====
    if (lane == 0 || (SPLIT_PRODUCER && lane == 1)) {
      int stage = 0; uint32_t phase = 0;
      for (int kbi = 0; kbi < pre; ++kbi) {                 // activation halves of the stages started above
        const int kb = kb_begin + kbi;
        const int tap = kb / kblocks_per_tap;
        const int kk = (kb - tap * kblocks_per_tap) * BK;
        tma_load_3d(smem + kbi * L::STAGE_BYTES, &map_a, &full_bar[kbi], kk, m0 + tap * ep.tap_dil - pad, bz * a_batch_mul);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      for (int kbi = pre; kbi < num_kb; ++kbi) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        const int kb = kb_begin + kbi;
        const int tap = kb / kblocks_per_tap;
        const int kk = (kb - tap * kblocks_per_tap) * BK;
        uint8_t* sa = smem + stage * L::STAGE_BYTES;
        uint8_t* sb = sa + L::A_BYTES;
        if constexpr (SPLIT_PRODUCER) {
          if (lane == 0) {
            mbar_arrive_expect_tx(&full_bar[stage], L::A_BYTES);
            tma_load_3d(sa, &map_a, &full_bar[stage], kk, m0 + tap * ep.tap_dil - pad, bz * a_batch_mul);
          } else {
            mbar_arrive_expect_tx(&full_bar[stage], L::B_BYTES);
            tma_load_3d(sb, &map_b, &full_bar[stage], tap * K + kk, n0, 0);
          }
        } else {
          mbar_arrive_expect_tx(&full_bar[stage], L::STAGE_BYTES);
          tma_load_3d(sa, &map_a, &full_bar[stage], kk, m0 + tap * ep.tap_dil - pad, bz * a_batch_mul);
          tma_load_3d(sb, &map_b, &full_bar[stage], tap * K + kk, n0, 0);
        }
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
    __syncwarp();
    pdl_launch_dependents();      // PDL trigger at the TAIL: the dependents' CTAs may be scheduled once every CTA of this
                                  // grid has all its loads in flight
  } else {
    // ===== consumers: warpgroup wg owns accumulator rows [64 wg, 64 wg + 64); then the epilogue =====
    const int wg = warp >> 2;
    const int rb = warp >> 1;                         // 32-row block this warp finishes in the epilogue
    if (ep.residual) {
      // pull the tile's residual rows into L2 ahead of the epilogue
      const int m = m0 + rb * 32 + lane;
      if (m < M && !(warp & 1)) {
        const float* p = ep.residual + (long long)bz * ep.res_bstride + (long long)m * ep.ldr + n0;
#pragma unroll
        for (int c = 0; c < BN; c += 32)
          if (n0 + c < N) asm volatile("prefetch.global.L2 [%0];" ::"l"(p + c));
      }
    }
    float acc[BN / 2];
    int stage = 0; uint32_t phase = 0;
    if (tr && threadIdx.x == 0) tr[3] = global_timer_ns();
    gemm_consumer_mainloop<BN, STAGES>(acc, smem, L::STAGE_BYTES, L::A_BYTES, full_bar, empty_bar, num_kb, stage, phase, wg,
                                       (threadIdx.x & 127) == 0, [](uint64_t* b) { mbar_arrive(b); });
    if (tr && threadIdx.x == 0) tr[4] = global_timer_ns();
    pdl_launch_dependents();
    // every wgmma of both warpgroups has retired: the pipeline stages are idle and take the staged accumulator tile
    named_barrier(1, GEMM_CONSUMERS);
    gemm_stage_accumulator<BN>(acc, smem_u32(smem), warp, lane);
    named_barrier(1, GEMM_CONSUMERS);
    if (tr && threadIdx.x == 0) tr[5] = global_timer_ns();
    gemm_epilogue_dispatch<BN>(smem_u32(smem) + (uint32_t)(rb * 32 * (BN + 8)) * 4, n0, N, m0 + rb * 32, M, lane, (long long)bz,
                               ep, warp & 1, 2);
    if (tr && threadIdx.x == 0) tr[6] = global_timer_ns();
  }
  __syncthreads();
  if (tr && threadIdx.x == 0) tr[7] = global_timer_ns();
}

// ------------------------------------------------------------------ reference (SIMT) GEMM: test/bring-up checker
__global__ void gemm_ref_kernel(const __nv_bfloat16* A, long long a_bstride, int lda, int rows, const __nv_bfloat16* W,
                                int M, int N, int K, int taps, int pad, GemmEpilogue ep) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  const int m = blockIdx.y;
  const int bz = blockIdx.z;
  if (n >= N || m >= M) return;
  const int nn = (ep.act == TTB_ACT_GEGLU) ? (n & ~1) : n;
  float acc[2] = {0.f, 0.f};
  const int cnt = (ep.act == TTB_ACT_GEGLU) ? 2 : 1;
  if (ep.act == TTB_ACT_GEGLU && (n & 1)) return;
  for (int c = 0; c < cnt; ++c) {
    float s = 0.f;
    for (int tap = 0; tap < taps; ++tap) {
      const int r = m + tap - pad;
      if (r < 0 || r >= rows) continue;
      const __nv_bfloat16* a = A + (long long)bz * a_bstride + (long long)r * lda;
      const __nv_bfloat16* w = W + (long long)(nn + c) * taps * K + (long long)tap * K;
      for (int k = 0; k < K; ++k) s += __bfloat162float(a[k]) * __bfloat162float(w[k]);
    }
    s *= ep.alpha;
    if (ep.bias) s += ep.bias[nn + c];
    acc[c] = s;
  }
  float v;
  int on = n;
  if (ep.act == TTB_ACT_GEGLU) { v = acc[0] * gelu_erf(acc[1]); on = n >> 1; }
  else {
    v = acc[0];
    if (ep.act == TTB_ACT_GELU_NEW) v = gelu_new(v);
    else if (ep.act == TTB_ACT_SILU) v = silu(v);
    else if (ep.act == TTB_ACT_LRELU02) v = leaky(v, 0.2f);
    else if (ep.act == TTB_ACT_GELU_ERF) v = gelu_erf(v);
    if (ep.residual) v += ep.residual[(long long)bz * ep.res_bstride + (long long)m * ep.ldr + n];
  }
  if (ep.out_f32) ep.out_f32[(long long)bz * ep.outf_bstride + (long long)m * ep.ldo + on] = v;
  if (ep.out_bf16) ep.out_bf16[(long long)bz * ep.outb_bstride + (long long)m * ep.ldob + on] = __float2bfloat16(v);
}

static unsigned long long* g_gemm_trace = nullptr;   // ttb_debug_gemm_trace

template <int BN, int STAGES, bool SPLIT_PRODUCER = false>
static int launch_tc(const TtbGemmArgs& g, const GemmEpilogue& ep, cudaStream_t st) {
  CUtensorMap ma, mb;
  // a_bstride == 0 broadcasts one activation tensor to every batch item (batch dim of extent 1, coordinate 0)
  const bool bcast = (g.batch == 1) || (g.a_bstride == 0);
  const uint64_t a_d2 = bcast ? 1 : (uint64_t)g.batch;
  const uint64_t a_s2 = bcast ? (uint64_t)g.rows * g.lda : (uint64_t)g.a_bstride;
  if (get_tensor_map_bf16(&ma, g.A, (uint64_t)g.K, (uint64_t)g.rows, a_d2, (uint64_t)g.lda, a_s2, BK, BM)) return -1;
  if (get_tensor_map_bf16(&mb, g.W, (uint64_t)g.K * g.taps, (uint64_t)g.N, 1, (uint64_t)g.K * g.taps,
                          (uint64_t)g.K * g.taps * g.N, BK, BN)) return -1;
  using L = GemmSmem<BN, STAGES>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gemm_bf16_tc_kernel<BN, STAGES, SPLIT_PRODUCER>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL);
    if (e != cudaSuccess) return check_cuda(e, "cudaFuncSetAttribute(gemm)");
    attr_set = true;
  }
  int kb_per_split = 0, zdim = g.batch;
  if (g.splitk > 1) {
    const int kb_total = (g.K / BK) * g.taps;
    kb_per_split = (kb_total + g.splitk - 1) / g.splitk;
    zdim = (kb_total + kb_per_split - 1) / kb_per_split;     // every split owns >= 1 k-block
  }
  dim3 grid((g.N + BN - 1) / BN, (g.M + BM - 1) / BM, zdim);
  cudaError_t le = launch_pdl(gemm_bf16_tc_kernel<BN, STAGES, SPLIT_PRODUCER>, grid, dim3(GEMM_THREADS), (size_t)L::TOTAL, st, ma, mb, g.M, g.N,
                              g.K, g.taps, g.pad, (bcast || g.splitk > 1) ? 0 : 1, kb_per_split, ep, g_gemm_trace);
  if (le != cudaSuccess) return check_cuda(le, "gemm_bf16_tc_kernel launch");
  TTB_CHECK_LAUNCH("gemm_bf16_tc_kernel");
  return 0;
}

}  // namespace ttb

#include "gemm_persist.cuh"
#include "gemm_mc.cuh"
#include "gemm_ws.cuh"

namespace ttb {

static int num_sms() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

template <int BN, int PSTAGES>
static int launch_persistent(const TtbGemmArgs& g, const GemmEpilogue& ep, cudaStream_t st) {
  CUtensorMap ma, mb;
  const bool bcast = (g.batch == 1) || (g.a_bstride == 0);
  const uint64_t a_d2 = bcast ? 1 : (uint64_t)g.batch;
  const uint64_t a_s2 = bcast ? (uint64_t)g.rows * g.lda : (uint64_t)g.a_bstride;
  if (get_tensor_map_bf16(&ma, g.A, (uint64_t)g.K, (uint64_t)g.rows, a_d2, (uint64_t)g.lda, a_s2, BK, BM)) return -1;
  if (get_tensor_map_bf16(&mb, g.W, (uint64_t)g.K * g.taps, (uint64_t)g.N, 1, (uint64_t)g.K * g.taps,
                          (uint64_t)g.K * g.taps * g.N, BK, BN)) return -1;
  using L = GemmPSmem<BN, PSTAGES>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gemm_bf16_tc_persistent_kernel<BN, PSTAGES>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL);
    if (e != cudaSuccess) return check_cuda(e, "cudaFuncSetAttribute(gemm persistent)");
    attr_set = true;
  }
  int kb_per_split = 0, zdim = g.batch;
  if (g.splitk > 1) {
    const int kb_total = (g.K / BK) * g.taps;
    kb_per_split = (kb_total + g.splitk - 1) / g.splitk;
    zdim = (kb_total + kb_per_split - 1) / kb_per_split;
  }
  const int m_tiles = (g.M + BM - 1) / BM, n_tiles = (g.N + BN - 1) / BN;
  const long long total = (long long)m_tiles * n_tiles * zdim;
  const int grid = (int)(total < num_sms() ? total : num_sms());
  const cudaError_t le = launch_pdl(gemm_bf16_tc_persistent_kernel<BN, PSTAGES>, dim3(grid), dim3(GEMM_THREADS), (size_t)L::TOTAL, st,
      ma, mb, g.M, g.N, g.K, g.taps, g.pad, (bcast || g.splitk > 1) ? 0 : 1, kb_per_split, m_tiles, n_tiles, zdim, ep);
  if (le != cudaSuccess) return check_cuda(le, "gemm_bf16_tc_persistent_kernel launch");
  TTB_CHECK_LAUNCH("gemm_bf16_tc_persistent_kernel");
  return 0;
}

// Persistent warp-specialised 128x256 kernel (gemm_ws.cuh): one CTA per SM, or one per tile when there are fewer.
static int launch_ws(const TtbGemmArgs& g, const GemmEpilogue& ep, cudaStream_t st) {
  CUtensorMap ma, mb;
  const bool bcast = (g.batch == 1) || (g.a_bstride == 0);
  const uint64_t a_d2 = bcast ? 1 : (uint64_t)g.batch;
  const uint64_t a_s2 = bcast ? (uint64_t)g.rows * g.lda : (uint64_t)g.a_bstride;
  if (get_tensor_map_bf16(&ma, g.A, (uint64_t)g.K, (uint64_t)g.rows, a_d2, (uint64_t)g.lda, a_s2, BK, BM)) return -1;
  if (get_tensor_map_bf16(&mb, g.W, (uint64_t)g.K * g.taps, (uint64_t)g.N, 1, (uint64_t)g.K * g.taps,
                          (uint64_t)g.K * g.taps * g.N, BK, WS_BN)) return -1;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gemm_bf16_ws_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, GemmWsSmem::TOTAL);
    if (e != cudaSuccess) return check_cuda(e, "cudaFuncSetAttribute(gemm ws)");
    attr_set = true;
  }
  const int m_tiles = (g.M + BM - 1) / BM, n_tiles = (g.N + WS_BN - 1) / WS_BN;
  const long long total = (long long)m_tiles * n_tiles * g.batch;
  const int grid = (int)(total < num_sms() ? total : num_sms());
  const cudaError_t le = launch_pdl(gemm_bf16_ws_kernel, dim3(grid), dim3(WS_THREADS), (size_t)GemmWsSmem::TOTAL, st,
      ma, mb, g.M, g.N, g.K, g.taps, g.pad, bcast ? 0 : 1, m_tiles, n_tiles, g.batch, ep);
  if (le != cudaSuccess) return check_cuda(le, "gemm_bf16_ws_kernel launch");
  TTB_CHECK_LAUNCH("gemm_bf16_ws_kernel");
  return 0;
}

}  // namespace ttb

using namespace ttb;

extern "C" int ttb_debug_gemm_trace(void* buf) {
  g_gemm_trace = static_cast<unsigned long long*>(buf);
  return 0;
}

extern "C" int ttb_gemm(const TtbGemmArgs* gp, void* stream) {
  const TtbGemmArgs& g = *gp;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (g.K % BK != 0 || g.K <= 0) { set_error("ttb_gemm: K=%d must be a positive multiple of 64", g.K); return -1; }
  if (g.taps < 1 || g.M <= 0 || g.N <= 0 || g.batch <= 0) { set_error("ttb_gemm: bad shape"); return -1; }
  if (g.act == TTB_ACT_GEGLU && (g.N & 1)) { set_error("ttb_gemm: GEGLU needs even N"); return -1; }
  GemmEpilogue ep;
  ep.bias = g.bias; ep.residual = g.residual; ep.out_f32 = g.out_f32;
  ep.out_bf16 = reinterpret_cast<__nv_bfloat16*>(g.out_bf16);
  ep.res_bstride = g.res_bstride; ep.outf_bstride = g.outf_bstride; ep.outb_bstride = g.outb_bstride;
  ep.ldr = g.ldr; ep.ldo = g.ldo; ep.ldob = g.ldob; ep.act = g.act; ep.alpha = g.alpha;
  ep.gn_part = nullptr; ep.gn_groups = g.gn_groups;
  ep.wpre = g.w_static;
  ep.tap_dil = g.tap_dilation > 1 ? g.tap_dilation : 1;
  if (ep.tap_dil > 1 && (g.cluster > 1 || g.variant == 6 || g.force_ref)) {
    set_error("ttb_gemm: tap_dilation is implemented by the one-tile and the persistent kernels only");
    return -1;
  }
  if (g.gn_partials) {
    if (g.N != 32 * g.gn_groups || (g.M + 31) / 32 > TTB_GN_SPLITS || g.act == TTB_ACT_GEGLU || g.splitk > 1 || g.force_ref) {
      set_error("ttb_gemm: gn_partials needs N == 32 * gn_groups, M <= %d, no GEGLU / split-K (N=%d groups=%d M=%d)",
                32 * TTB_GN_SPLITS, g.N, g.gn_groups, g.M);
      return -1;
    }
    ep.gn_part = reinterpret_cast<float2*>(g.gn_partials + 16);   // scratch layout of norm.cu: 16 floats, then the partials
  }
  if (g.splitk > 1) {
    // split-K writes raw fp32 partials [split, M, ldo] (consumed by ttb_residual_layernorm); no epilogue fusion
    if (g.batch != 1 || g.act != TTB_ACT_NONE || !g.out_f32 || g.out_bf16 || g.bias || g.residual) {
      set_error("ttb_gemm: splitk needs batch=1, no activation/bias/residual and an fp32 partial buffer");
      return -1;
    }
    if (g.force_ref) { set_error("ttb_gemm: splitk is not available in the SIMT checker"); return -1; }
  }
  if (g.force_ref) {
    dim3 block(128), grid((g.N + 127) / 128, g.M, g.batch);
    gemm_ref_kernel<<<grid, block, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(g.A), g.a_bstride, g.lda, g.rows,
                                            reinterpret_cast<const __nv_bfloat16*>(g.W), g.M, g.N, g.K, g.taps, g.pad, ep);
    TTB_CHECK_LAUNCH("gemm_ref_kernel");
    return 0;
  }
  // tile choice: fill the SMs; small-N / small-M problems use narrower tiles
  const long long tiles128 = (long long)((g.N + 127) / 128) * ((g.M + BM - 1) / BM) * g.batch;
  if (g.cluster > 1) {
    // thread-block clusters along N sharing the activation tile by TMA multicast (gemm_mc.cuh)
    const int bn = g.tile_n == 32 ? 32 : (g.tile_n == 64 ? 64 : 128);
    const int n_tiles = (g.N + bn - 1) / bn;
    if ((g.cluster != 2 && g.cluster != 4) || n_tiles % g.cluster != 0) {
      set_error("ttb_gemm: cluster=%d needs 2 or 4 and a multiple of it in N tiles (%d)", g.cluster, n_tiles);
      return -1;
    }
    if (bn == 32) return g.cluster == 4 ? launch_mc<32, 4, 4>(g, ep, st) : launch_mc<32, 4, 2>(g, ep, st);
    if (bn == 64) return g.cluster == 4 ? launch_mc<64, 4, 4>(g, ep, st) : launch_mc<64, 4, 2>(g, ep, st);
    return g.cluster == 4 ? launch_mc<128, 3, 4>(g, ep, st) : launch_mc<128, 3, 2>(g, ep, st);
  }
  if (g.variant == 6) { set_error("ttb_gemm: variant 6 (CTA-pair MMA) needs hardware this library does not target"); return -1; }
  if (g.variant == 7) {
    if (g.splitk > 1) { set_error("ttb_gemm: variant 7 (warp-specialised 128x256) has no split-K"); return -1; }
    return launch_ws(g, ep, st);
  }
  // The persistent 128x128 kernel only on request: on H100 (80GB HBM3, 700 W) the one-tile kernel was faster on every
  // stage that has several tiles per SM (standard preset: CLVP 156 -> 118 ms, diffusion 1061 -> 992 ms).
  if (g.variant == 2) {
    if (g.tile_n == 32) return launch_persistent<32, 8>(g, ep, st);
    if (g.tile_n == 64) return launch_persistent<64, 6>(g, ep, st);
    return launch_persistent<128, 4>(g, ep, st);
  }
  // Default for problems of at least one wave of 128x128 tiles: the persistent warp-specialised 128x256 kernel
  // (gemm_ws.cuh). variant 1 keeps the one-tile 128x128 kernel.
  if (g.tile_n == 0 && g.variant == 0 && g.splitk <= 1 && tiles128 >= num_sms()) return launch_ws(g, ep, st);
  if (g.tile_n == 32) {
    // the skinny decode GEMMs are latency-bound (k-block time = TMA round trip / stages): 5 stages still allow two
    // CTAs per SM (2 x 101 KB of the 227 KB). variant 4 selects the 4-stage kernel.
    return g.variant == 4 ? launch_tc<32, 4>(g, ep, st) : launch_tc<32, 5>(g, ep, st);
  }
  // 64-wide tiles, 8 stages, one CTA per SM (variant 3): for skinny problems whose 64-wide grid fits one wave, the deep
  // pipeline keeps ~190 KB in flight per SM
  if (g.tile_n == 64 && g.variant == 3) return launch_tc<64, 8>(g, ep, st);
  if (g.tile_n == 64 || (g.tile_n == 0 && tiles128 < num_sms())) return launch_tc<64, 4>(g, ep, st);
  // 128x256 tiles (64 vs 85 flop per operand byte) only on request
  if (g.tile_n == 256) return launch_tc<256, 3>(g, ep, st);
  if (g.variant == 5) return launch_tc<128, 3, true>(g, ep, st);     // two TMA issuers (experiment)
  return launch_tc<128, 3>(g, ep, st);
}
