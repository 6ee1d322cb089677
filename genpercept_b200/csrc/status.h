// The library's one error type and the one place a failure becomes a gp_status and a reason at the C-ABI.
#pragma once
#include <cuda_runtime.h>

#include <exception>
#include <string>
#include <utility>

#include "../../include/genpercept_b200.h"

namespace gp {

// A failure with the status its C-ABI call returns; what() is the reason the caller reads back.
struct GpError : std::exception {
  gp_status st;
  std::string msg;
  GpError(gp_status s, std::string m) : st(s), msg(std::move(m)) {}
  const char* what() const noexcept override { return msg.c_str(); }
};
#define GP_CUDA(call)                                                                           \
  do {                                                                                          \
    cudaError_t e__ = (call);                                                                   \
    if (e__ != cudaSuccess)                                                                     \
      throw ::gp::GpError(GP_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e__));    \
  } while (0)
#define GP_REQUIRE(cond, msg)                                             \
  do {                                                                    \
    if (!(cond)) throw ::gp::GpError(GP_ERR_INVALID, std::string(msg));   \
  } while (0)

// Runs `f`.  A GpError returns its own status, any other exception GP_ERR_INVALID; either way `err` gets its what().
// `err` is left alone on success.
template <class F>
gp_status run_guarded(F&& f, std::string& err) {
  try {
    f();
    return GP_OK;
  } catch (const GpError& ex) {
    err = ex.what();
    return ex.st;
  } catch (const std::exception& ex) {
    err = ex.what();
    return GP_ERR_INVALID;
  }
}

// The reason of the calling thread's last failed engine-free call, "" after a successful one (gp_last_call_error).
inline std::string& call_error() {
  static thread_local std::string s;
  return s;
}

// The guard of every C-ABI call that takes no engine.
template <class F>
gp_status guarded_call(F&& f) {
  call_error().clear();
  return run_guarded(f, call_error());
}

}  // namespace gp
