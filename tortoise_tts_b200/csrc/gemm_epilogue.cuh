// GEMM epilogue shared by the wgmma GEMM kernels (included by gemm.cu after GemmEpilogue is defined).
//
// wgmma leaves the accumulator spread over the registers of the two consumer warpgroups (8 rows x 4 column pairs per
// warp and instruction fragment). Writing fragments straight to global memory would touch 8 cache lines per store, so
// the tile first goes, raw, to a padded fp32 tile in shared memory (gemm_stage_accumulator); the epilogue then reads it
// back row-wise: 8 lanes cover one row's 128 bytes and a warp instruction moves 4 complete rows, for the residual read
// and the fp32 / bf16 writes alike. Each warp finishes one 32-row block, the two warps of a block alternate 32-column
// chunks.
//   * the activation is a template parameter and the run-time switch sits OUTSIDE the chunk loop;
//   * a chunk that is complete (32 columns, 16-byte aligned rows) takes a branch-free FAST path; ragged edges take a
//     separate, simple per-row SLOW path (lane = row);
//   * the residual (which may alias the output: x += f(x) in place) is loaded for the whole chunk before any store;
//   * the tile pitch is BN + 8 floats, so both the fragment stores and the row reads are conflict-free.
#pragma once

namespace ttb {

TTB_DEVINL float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
  return v;
}

// Accumulator fragments of this thread (rows 64 wg + 16 w + l/4 (+8), see common.cuh) -> fp32 tile [128][BN + 8].
template <int BN>
TTB_DEVINL void gemm_stage_accumulator(const float* acc, uint32_t tile, int cwarp, int lane) {
  constexpr int PITCH = BN + 8;
  const uint32_t base = tile + (uint32_t)((cwarp * 16 + (lane >> 2)) * PITCH + 2 * (lane & 3)) * 4;
#pragma unroll
  for (int i = 0; i < BN / 2; i += 4) {
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(base + (uint32_t)(2 * i) * 4), "f"(acc[i]), "f"(acc[i + 1]) : "memory");
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(base + (uint32_t)(8 * PITCH + 2 * i) * 4), "f"(acc[i + 2]), "f"(acc[i + 3]) : "memory");
  }
}

template <int ACT>
TTB_DEVINL float epi_act(float x) {
  if (ACT == TTB_ACT_GELU_NEW) return gelu_new(x);
  if (ACT == TTB_ACT_SILU) return silu(x);
  if (ACT == TTB_ACT_LRELU02) return leaky(x, 0.2f);
  if (ACT == TTB_ACT_TANH) return tanhf(x);
  if (ACT == TTB_ACT_GELU_ERF) return gelu_erf(x);
  return x;
}

// What a tile's epilogue needs to know once (warp-uniform).
struct EpiFlags {
  bool aligned;     // bias pointer, ldr, ldo, ldob all allow 128-bit (fp32) / 64-bit (bf16) row accesses
};

TTB_DEVINL EpiFlags epi_flags(const GemmEpilogue& ep) {
  EpiFlags f;
  f.aligned = (!ep.bias || (reinterpret_cast<uintptr_t>(ep.bias) & 15) == 0) &&
              (!ep.residual || ((ep.ldr & 3) == 0 && (ep.res_bstride & 3) == 0 && (reinterpret_cast<uintptr_t>(ep.residual) & 15) == 0)) &&
              (!ep.out_f32 || ((ep.ldo & 3) == 0 && (ep.outf_bstride & 3) == 0 && (reinterpret_cast<uintptr_t>(ep.out_f32) & 15) == 0)) &&
              (!ep.out_bf16 || ((ep.ldob & 3) == 0 && (ep.outb_bstride & 3) == 0 && (reinterpret_cast<uintptr_t>(ep.out_bf16) & 7) == 0));
  return f;
}

// (sum, sum of squares) of one 32-row x 32-column block of the output = one GroupNorm partial (32 channels per group):
// fixed xor tree, one writer, no atomics (bit-reproducible).
TTB_DEVINL void epi_gn_store(float gs, float gq, int nb, int m_base, int lane, long long bz, const GemmEpilogue& ep) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    gs += __shfl_xor_sync(0xffffffffu, gs, off);
    gq += __shfl_xor_sync(0xffffffffu, gq, off);
  }
  if (lane == 0)
    ep.gn_part[((long long)bz * ep.gn_groups + (nb >> 5)) * TTB_GN_SPLITS + (m_base >> 5)] = make_float2(gs, gq);
}

// ---- FAST path: all 32 columns exist, everything aligned. Branch-free apart from the uniform pointer tests. Only the
// first `rows_valid` (1..32) of the 32 rows exist (< 32: the last row block of a ragged M): the row-wise residual loads
// and stores are predicated per row. `blk` = shared-memory address of (first row of the block, first column of the
// chunk) in the staged accumulator tile, `pitch` in floats.
template <int ACT>
TTB_DEVINL void epi_chunk_fast(uint32_t blk, int pitch, int nb, int m_base, int rows_valid, int lane, long long bz,
                               const GemmEpilogue& ep) {
  const bool GN = ep.gn_part != nullptr;
  const int rr0 = lane >> 3, c = (lane & 7) * 4;     // 4 rows per instruction: 8 lanes x 4 columns per row
  float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
  if (ep.bias) b = __ldg(reinterpret_cast<const float4*>(ep.bias + nb + c));
  if (ACT == TTB_ACT_GEGLU) {
    // columns interleaved (u0,g0,u1,g1,...): out[j] = u * gelu_erf(g); output width N/2 -> 2 columns per lane
    const long long col = (nb >> 1) + (c >> 1);
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const int rr = it * 4 + rr0;
      const float4 a = lds128(blk + (uint32_t)(rr * pitch + c) * 4);
      const float o0 = fmaf(a.x, ep.alpha, b.x) * gelu_erf(fmaf(a.y, ep.alpha, b.y));
      const float o1 = fmaf(a.z, ep.alpha, b.z) * gelu_erf(fmaf(a.w, ep.alpha, b.w));
      const long long m = m_base + rr;
      if (rr >= rows_valid) continue;
      if (ep.out_bf16) *reinterpret_cast<uint32_t*>(ep.out_bf16 + bz * ep.outb_bstride + m * ep.ldob + col) = pack_bf16(o0, o1);
      if (ep.out_f32) *reinterpret_cast<float2*>(ep.out_f32 + bz * ep.outf_bstride + m * ep.ldo + col) = make_float2(o0, o1);
    }
    return;
  }
  const long long col = nb + c;
  // residual for the positions this lane stores, all issued before the first store
  float4 rs[8];
  if (ep.residual) {
    const float* rp = ep.residual + bz * ep.res_bstride + (long long)(m_base + rr0) * ep.ldr + col;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      if (it * 4 + rr0 < rows_valid) rs[it] = *reinterpret_cast<const float4*>(rp + (long long)it * 4 * ep.ldr);
      else rs[it] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  float gs = 0.f, gq = 0.f;                          // GroupNorm partial of this 32 x 32 block (ep.gn_part)
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int rr = it * 4 + rr0;
    const float4 a = lds128(blk + (uint32_t)(rr * pitch + c) * 4);
    float4 o;
    o.x = epi_act<ACT>(fmaf(a.x, ep.alpha, b.x));
    o.y = epi_act<ACT>(fmaf(a.y, ep.alpha, b.y));
    o.z = epi_act<ACT>(fmaf(a.z, ep.alpha, b.z));
    o.w = epi_act<ACT>(fmaf(a.w, ep.alpha, b.w));
    if (ep.residual) { o.x += rs[it].x; o.y += rs[it].y; o.z += rs[it].z; o.w += rs[it].w; }
    const long long m = m_base + rr;
    if (rr >= rows_valid) continue;
    if (ep.out_f32) *reinterpret_cast<float4*>(ep.out_f32 + bz * ep.outf_bstride + m * ep.ldo + col) = o;
    if (ep.out_bf16)
      *reinterpret_cast<uint2*>(ep.out_bf16 + bz * ep.outb_bstride + m * ep.ldob + col) = make_uint2(pack_bf16(o.x, o.y), pack_bf16(o.z, o.w));
    if (GN) {
      gs += (o.x + o.y) + (o.z + o.w);
      gq += (o.x * o.x + o.y * o.y) + (o.z * o.z + o.w * o.w);
    }
  }
  if (GN) epi_gn_store(gs, gq, nb, m_base, lane, bz, ep);
}

// ---- SLOW path (ragged M / N edges, unaligned rows): each lane finishes its own accumulator row with scalar accesses.
template <int ACT>
TTB_DEVINL void epi_chunk_slow(const uint32_t* r, int nb, int N, int m, int M, long long bz, const GemmEpilogue& ep,
                               float& gs, float& gq) {
  if (m >= M) return;
  if (ACT == TTB_ACT_GEGLU) {
    const int nout = N >> 1, ob = nb >> 1;
    float* of = ep.out_f32 ? ep.out_f32 + bz * ep.outf_bstride + (long long)m * ep.ldo : nullptr;
    __nv_bfloat16* obf = ep.out_bf16 ? ep.out_bf16 + bz * ep.outb_bstride + (long long)m * ep.ldob : nullptr;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      if (ob + j < nout) {
        float u = __uint_as_float(r[2 * j]) * ep.alpha, g = __uint_as_float(r[2 * j + 1]) * ep.alpha;
        if (ep.bias) { u += __ldg(ep.bias + nb + 2 * j); g += __ldg(ep.bias + nb + 2 * j + 1); }
        const float o = u * gelu_erf(g);
        if (of) of[ob + j] = o;
        if (obf) obf[ob + j] = __float2bfloat16(o);
      }
    }
    return;
  }
  const float* rp = ep.residual ? ep.residual + bz * ep.res_bstride + (long long)m * ep.ldr : nullptr;
  float* of = ep.out_f32 ? ep.out_f32 + bz * ep.outf_bstride + (long long)m * ep.ldo : nullptr;
  __nv_bfloat16* obf = ep.out_bf16 ? ep.out_bf16 + bz * ep.outb_bstride + (long long)m * ep.ldob : nullptr;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    if (nb + j < N) {
      float x = __uint_as_float(r[j]) * ep.alpha;
      if (ep.bias) x += __ldg(ep.bias + nb + j);
      x = epi_act<ACT>(x);
      if (rp) x += rp[nb + j];
      if (of) of[nb + j] = x;
      if (obf) obf[nb + j] = __float2bfloat16(x);
      gs += x;
      gq += x * x;
    }
  }
}

// One 32-row block of the staged accumulator tile, finished by one warp: `blk` = shared-memory address of the block's
// first row, chunks ch_begin, ch_begin + ch_step, ... of 32 columns.
template <int BN, int ACT>
TTB_DEVINL void gemm_epilogue_tile(uint32_t blk, int n0, int N, int m_base, int M, int lane, long long bz,
                                   const GemmEpilogue& ep, int ch_begin, int ch_step) {
  constexpr int NCH = BN / 32;
  constexpr int PITCH = BN + 8;
  const bool aligned = epi_flags(ep).aligned;
  const int rows_valid = min(32, M - m_base);        // warp-uniform; <= 0: this warp's rows are all past M
  // rolled on purpose: one chunk's worth of code and registers
#pragma unroll 1
  for (int ch = ch_begin; ch < NCH; ch += ch_step) {
    const int nb = n0 + ch * 32;
    if (nb >= N || rows_valid <= 0) continue;        // warp-uniform
    if (aligned && nb + 32 <= N) {
      epi_chunk_fast<ACT>(blk + (uint32_t)ch * 128, PITCH, nb, m_base, rows_valid, lane, bz, ep);
    } else {
      uint32_t r[32];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 a = lds128(blk + (uint32_t)(lane * PITCH + ch * 32 + 4 * j) * 4);
        r[4 * j] = __float_as_uint(a.x); r[4 * j + 1] = __float_as_uint(a.y);
        r[4 * j + 2] = __float_as_uint(a.z); r[4 * j + 3] = __float_as_uint(a.w);
      }
      float gs = 0.f, gq = 0.f;                      // rows past M contribute nothing
      epi_chunk_slow<ACT>(r, nb, N, m_base + lane, M, bz, ep, gs, gq);
      if (ep.gn_part) epi_gn_store(gs, gq, nb, m_base, lane, bz, ep);
    }
  }
}

template <int BN>
TTB_DEVINL void gemm_epilogue_dispatch(uint32_t blk, int n0, int N, int m_base, int M, int lane, long long bz,
                                       const GemmEpilogue& ep, int ch_begin, int ch_step) {
  switch (ep.act) {
    case TTB_ACT_GEGLU: gemm_epilogue_tile<BN, TTB_ACT_GEGLU>(blk, n0, N, m_base, M, lane, bz, ep, ch_begin, ch_step); break;
    case TTB_ACT_GELU_NEW: gemm_epilogue_tile<BN, TTB_ACT_GELU_NEW>(blk, n0, N, m_base, M, lane, bz, ep, ch_begin, ch_step); break;
    case TTB_ACT_SILU: gemm_epilogue_tile<BN, TTB_ACT_SILU>(blk, n0, N, m_base, M, lane, bz, ep, ch_begin, ch_step); break;
    case TTB_ACT_LRELU02: gemm_epilogue_tile<BN, TTB_ACT_LRELU02>(blk, n0, N, m_base, M, lane, bz, ep, ch_begin, ch_step); break;
    case TTB_ACT_TANH: gemm_epilogue_tile<BN, TTB_ACT_TANH>(blk, n0, N, m_base, M, lane, bz, ep, ch_begin, ch_step); break;
    case TTB_ACT_GELU_ERF: gemm_epilogue_tile<BN, TTB_ACT_GELU_ERF>(blk, n0, N, m_base, M, lane, bz, ep, ch_begin, ch_step); break;
    default: gemm_epilogue_tile<BN, TTB_ACT_NONE>(blk, n0, N, m_base, M, lane, bz, ep, ch_begin, ch_step); break;
  }
}

}  // namespace ttb
