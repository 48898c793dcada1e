// Internal declarations shared by the .cu files of libttb.so
#pragma once
#include "../../include/ttb.h"
#include <cuda_runtime.h>
#include <cuda.h>
#include <cstdlib>

#define TTB_GN_SPLITS TTB_GROUPNORM_SPLITS   // row blocks of the GroupNorm statistics pass (include/ttb.h)

namespace ttb {
// flash_attn.cu: wgmma attention for the large shapes
bool flash_attention_supported(const TtbAttnArgs& a);
int flash_attention_launch(const TtbAttnArgs& a, cudaStream_t st);
// gemm.cu
int get_tensor_map_bf16(CUtensorMap* out, const void* ptr, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t stride1_elems,
                        uint64_t stride2_elems, uint32_t b0, uint32_t b1);
int make_tensor_map_bf16_nd(CUtensorMap* out, const void* ptr, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                            const uint32_t* box);
}
