// Common device helpers for the tortoise-b200 kernels (sm_90a only).
// PTX wrappers: mbarrier, TMA (cp.async.bulk.tensor), wgmma (fence / mma_async / commit / wait), fences.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda.h>
#include <stdint.h>
#include <cstdlib>

#define TTB_DEVINL __device__ __forceinline__

namespace ttb {

// ------------------------------------------------------------------ error plumbing (host)
void set_error(const char* fmt, ...);
int check_cuda(cudaError_t e, const char* what);
#define TTB_CHECK_LAUNCH(what)                                   \
  do {                                                           \
    cudaError_t _e = cudaGetLastError();                         \
    if (_e != cudaSuccess) return ttb::check_cuda(_e, what);     \
  } while (0)

// ------------------------------------------------------------------ programmatic dependent launch (PDL)
// Every kernel of the two per-step CUDA graphs starts with pdl_launch_dependents() and calls pdl_wait() before its
// first access to global memory that an earlier kernel may have written (and before its own first global write).
// Launched the ordinary way both instructions are no-ops. With TTB_PDL=1 the host launches these kernels with
// cudaLaunchAttributeProgrammaticStreamSerialization: the next kernel's CTAs are scheduled, run their prologue
// (barrier init, descriptor prefetch) and park in griddepcontrol.wait while the previous kernel drains, which removes
// the kernel-to-kernel launch gap that dominates the short decode-step kernels. The triggers sit at the kernels' TAILS
// (GEMM: once all loads of the CTA are issued and its accumulator is complete; LayerNorm: after its loads; others: at
// exit): a trigger at the top makes the dependent's CTAs resident at once, and they take registers / shared memory
// away from the kernel still running. On by default; TTB_PDL=0 restores plain launches.
TTB_DEVINL void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
TTB_DEVINL void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

inline bool pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("TTB_PDL");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  return v == 1;
}

// kernel<<<grid, block, smem, st>>>(args...) with the PDL launch attribute when TTB_PDL=1. Only for kernels that
// contain pdl_wait().
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  if (pdl_enabled()) {
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
  }
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// ------------------------------------------------------------------ small math
TTB_DEVINL float silu(float x) { return x / (1.0f + __expf(-x)); }
TTB_DEVINL float gelu_new(float x) {
  // HF NewGELUActivation: 0.5 x (1 + tanh(sqrt(2/pi) (x + 0.044715 x^3)))
  const float k = 0.7978845608028654f;
  float u = k * (x + 0.044715f * x * x * x);
  return 0.5f * x * (1.0f + tanhf(u));
}
TTB_DEVINL float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.7071067811865476f)); }
TTB_DEVINL float leaky(float x, float s) { return x > 0.f ? x : x * s; }

TTB_DEVINL float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
TTB_DEVINL float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// block-wide sum for blockDim.x <= 1024; `red` is >= 32 floats of shared memory
TTB_DEVINL float block_sum(float v, float* red) {
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  float r = (lane < nw) ? red[lane] : 0.f;
  r = warp_sum(r);
  return r;
}
TTB_DEVINL float block_max(float v, float* red) {
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_max(v);
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  float r = (lane < nw) ? red[lane] : -INFINITY;
  r = warp_max(r);
  return r;
}

TTB_DEVINL uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}
TTB_DEVINL float2 unpack_bf16(uint32_t u) {
  __nv_bfloat162 t = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(t);
}

TTB_DEVINL uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

TTB_DEVINL unsigned long long global_timer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
TTB_DEVINL unsigned long long sm_id() {
  uint32_t s;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(s));
  return s;
}

TTB_DEVINL bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t.reg .b32 R;\n\t"
      "elect.sync R|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ------------------------------------------------------------------ mbarrier
TTB_DEVINL void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
TTB_DEVINL void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
TTB_DEVINL void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
TTB_DEVINL void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
TTB_DEVINL void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// try_wait with a suspend-time hint: the waiting warp is parked by the hardware until the phase completes (or the hint
// expires) instead of re-issuing the poll every few cycles -- the polls of the waiting roles (epilogue warps during a
// mainloop, the single-lane TMA / MMA issuers) otherwise take issue slots from the warps doing the work on the same
// scheduler.
// TTB_MBAR_HINT_NS=0 at build time restores the plain poll loop (A/B).
#ifndef TTB_MBAR_HINT_NS
#define TTB_MBAR_HINT_NS 20000
#endif
TTB_DEVINL void mbar_wait(uint64_t* bar, uint32_t parity) {
#if TTB_MBAR_HINT_NS > 0
  asm volatile(
      "{\n\t.reg .pred P1;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1, %2;\n\t"
      "@P1 bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t}\n" ::"r"(smem_u32(bar)),
      "r"(parity), "r"((uint32_t)TTB_MBAR_HINT_NS)
      : "memory");
#else
  asm volatile(
      "{\n\t.reg .pred P1;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
#endif
}

// ------------------------------------------------------------------ TMA
TTB_DEVINL void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
TTB_DEVINL void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
TTB_DEVINL void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// L2 prefetch of one box of a 3-D tensor map (no shared-memory destination, no barrier)
TTB_DEVINL void tma_prefetch_l2_3d(const CUtensorMap* map, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.prefetch.tensor.3d.L2.global.tile [%0, {%1, %2, %3}];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}

// ------------------------------------------------------------------ wgmma (Hopper warpgroup MMA)
// A warpgroup = 4 consecutive warps whose first warp index is a multiple of 4. All 128 threads issue the instruction;
// the fp32 accumulator lives in their registers: for m64nN, register i of lane l of warp w holds
//   row = 16 w + l / 4 + 8 ((i >> 1) & 1),   column = 8 (i >> 2) + 2 (l & 3) + (i & 1).
TTB_DEVINL void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
TTB_DEVINL void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
TTB_DEVINL void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
TTB_DEVINL void named_barrier(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

// Shared-memory matrix descriptor (sm_90), K-major operand, SWIZZLE_128B, bf16:
//   rows of 64 elements (128 B), 8-row swizzle atoms of 1024 B (SBO = 1024), LBO ignored (=1), layout type 1 =
//   128-byte swizzle (bits 62-63). (cute::GmmaDescriptor, cute/arch/mma_sm90_desc.hpp)
TTB_DEVINL uint64_t wgmma_desc_kmajor_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);        // start address
  d |= (uint64_t)1 << 16;                             // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)(1024 >> 4) << 32;                   // stride byte offset: 8 rows * 128 B
  d |= (uint64_t)1 << 62;                             // SWIZZLE_128B
  return d;
}
// MN-major operand (e.g. V [keys, 64 dims] used as B[N=64 dims, K=keys], transposed by the instruction), SWIZZLE_128B:
//   64 MN-elements contiguous (128 B) per K index; 8 K-rows per 1024-B atom (SBO = 1024);
//   LBO = byte distance between 64-wide MN groups.
TTB_DEVINL uint64_t wgmma_desc_mnmajor_sw128(uint32_t smem_addr, uint32_t lbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// D[registers] (+)= A[smem] * B[smem]^T (both K-major); scale_d == 0 overwrites D.
TTB_DEVINL void wgmma_m64n16k16_bf16_ss(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d));
}
TTB_DEVINL void wgmma_m64n32k16_bf16_ss(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d));
}
TTB_DEVINL void wgmma_m64n64k16_bf16_ss(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d));
}
// 64 x 256 x 16 in one instruction: the A slice is read from shared memory once for all 256 columns (gemm_ws.cuh).
TTB_DEVINL void wgmma_m64n256k16_bf16_ss(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d));
}
// A from registers (the m16n8k16 A-fragment layout per warp), B from smem; TNSPB = 1: B is MN-major.
template <int TNSPB>
TTB_DEVINL void wgmma_m64n64k16_bf16_rs(float* d, const uint32_t* a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, %38;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(scale_d), "n"(TNSPB));
}

// The k-block of one consumer warpgroup: acc[64 x BN] (+)= A[64 rows x 64] * B[BN rows x 64]^T, both K-major SWIZZLE_128B
// tiles in shared memory (sa = this warpgroup's 64 rows). BN = 32: one n32 instruction per k16, else BN / 64 n64 ones.
template <int BN>
TTB_DEVINL void gemm_mma_kblock(float* acc, uint32_t sa, uint32_t sb, bool first) {
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const uint64_t da = wgmma_desc_kmajor_sw128(sa + k * 32);
    const uint32_t sc = (first && k == 0) ? 0u : 1u;
    if constexpr (BN == 32) {
      wgmma_m64n32k16_bf16_ss(acc, da, wgmma_desc_kmajor_sw128(sb + k * 32), sc);
    } else {
#pragma unroll
      for (int nb = 0; nb < BN / 64; ++nb)
        wgmma_m64n64k16_bf16_ss(acc + nb * 32, da, wgmma_desc_kmajor_sw128(sb + nb * 8192 + k * 32), sc);
    }
  }
  wgmma_commit();
}

// The k-block of one consumer warpgroup with a 256-wide B tile: one m64n256k16 per k16 step (same k order as
// gemm_mma_kblock, and the same accumulator layout as gemm_mma_kblock<256>: register i -> column 8 (i >> 2) + ...).
TTB_DEVINL void gemm_mma_kblock_n256(float* acc, uint32_t sa, uint32_t sb, bool first) {
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 4; ++k)
    wgmma_m64n256k16_bf16_ss(acc, wgmma_desc_kmajor_sw128(sa + k * 32), wgmma_desc_kmajor_sw128(sb + k * 32),
                             (first && k == 0) ? 0u : 1u);
  wgmma_commit();
}

// Warp-specialised kernels: a warpgroup that only issues TMA hands registers back to the pool, the MMA warpgroups take
// them (the counts are per thread, multiples of 8, and apply to all 128 threads of the executing warpgroup).
template <int R>
TTB_DEVINL void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
TTB_DEVINL void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }


}  // namespace ttb
