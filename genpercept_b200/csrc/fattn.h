// Fused (FlashAttention-style) self-attention forward for head_dim 64 on wgmma; see fattn.cu.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

namespace gp {

struct FattnParams {
  CUtensorMap tmQ;   // (C, T, B)  box (64, 128, 1) over the q part of the packed qk tensor
  CUtensorMap tmK;   // (C, T, B)  box (64, 128, 1) over the k part
  CUtensorMap tmV;   // (T, C, B)  box (64, 64, 1)  over V^T  [B][C][Tp]
  void* out;         // 16-bit [B, T, heads*64] (+ the lo plane at out_lo)
  long long out_b_stride;
  int out_row_stride;
  int T, heads, B, q_tiles;
  float scale_log2e;
  int bf16;
  // high-precision mode (split != 0, fp16): the lo planes of q, k and V^T, and the element offset of o's lo plane
  // inside an output row
  int split;
  int out_lo;
  CUtensorMap tmQl, tmKl, tmVl;
};

cudaError_t fattn_launch(const FattnParams& p, cudaStream_t stream);

}  // namespace gp
