// Fused (FlashAttention-style) single-head self-attention forward for head_dim 512 on wgmma; see fattn512.cu.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

namespace gp {

struct Fattn512Params {
  CUtensorMap tmQ;   // (512, T, B)  box (64, 64, 1) over the q half of the packed qk tensor
  CUtensorMap tmK;   // (512, T, B)  box (64, 64, 1) over the k half
  CUtensorMap tmV;   // (T, 512, B)  box (64, 64, 1) over V^T  [B][512][Tp]
  void* out;         // 16-bit [B, T, out_row_stride], columns 0..511 (+ the lo plane at out_lo)
  const float* bias; // [512] added to every output row (the to_v bias), or nullptr
  long long out_b_stride;
  int out_row_stride;
  int T, B, q_tiles;
  float scale_log2e;
  int bf16;
  // high-precision mode (split != 0, fp16): the lo planes of q, k and V^T, and the element offset of o's lo plane
  // inside an output row
  int split;
  int out_lo;
  CUtensorMap tmQl, tmKl, tmVl;
};

cudaError_t fattn512_launch(const Fattn512Params& p, cudaStream_t stream);

}  // namespace gp
