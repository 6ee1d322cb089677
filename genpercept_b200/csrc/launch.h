// Kernel launch helper: cudaLaunchKernelEx, optionally with the programmatic-dependent-launch attribute (see ptx.cuh,
// pdl_wait).  Opt-in (GP_PDL=1): inside a CUDA graph the launch gaps are already short and the early-resident CTAs
// only add scheduling work.
#pragma once
#include <cuda_runtime.h>

#include <cstdlib>

namespace gp {

inline bool pdl_enabled() {
  static const bool on = [] { const char* e = getenv("GP_PDL"); return e && e[0] == '1'; }();
  return on;
}

template <typename... P, typename... A>
inline cudaError_t launch(void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, A&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<P>(args)...);
}

}  // namespace gp
