// Kernel launch helper: the one launch idiom of the engine (cudaLaunchKernelEx with the kernel's argument types).
#pragma once
#include <cuda_runtime.h>

namespace gp {

template <typename... P, typename... A>
inline cudaError_t launch(void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, A&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<P>(args)...);
}

}  // namespace gp
