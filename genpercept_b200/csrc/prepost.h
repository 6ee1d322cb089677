// Shared state of the engine-free pre/post entry points (imgproc.cu, evaluate.cu): one lock, one growing device
// scratch buffer per device, and the error mapping of their C-ABI functions.
#pragma once
#include <cuda_runtime.h>
#include <stdio.h>

#include <mutex>
#include <stdexcept>
#include <string>

#include "../../include/genpercept_b200.h"

namespace gp {

std::mutex& prepost_mutex();
// Device scratch for `dev`, at least `bytes` long; it only grows.  Callers hold prepost_mutex() and use it stream-ordered.
void* prepost_scratch(int dev, size_t bytes);

inline void prepost_ck(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}

// std::invalid_argument -> GP_ERR_INVALID, any other exception -> GP_ERR_CUDA; the message goes to stderr.
template <typename F>
gp_status prepost_guarded(F f) {
  try {
    f();
    return GP_OK;
  } catch (const std::invalid_argument& ex) {
    fprintf(stderr, "[genpercept_b200] %s\n", ex.what());
    return GP_ERR_INVALID;
  } catch (const std::exception& ex) {
    fprintf(stderr, "[genpercept_b200] %s\n", ex.what());
    return GP_ERR_CUDA;
  }
}

}  // namespace gp
