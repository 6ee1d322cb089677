// Shared state of the engine-free pre/post entry points (imgproc.cu, evaluate.cu): one lock and one growing device
// scratch buffer per device.
#pragma once
#include <stddef.h>

#include <mutex>

namespace gp {

std::mutex& prepost_mutex();
// Device scratch for `dev`, at least `bytes` long; it only grows.  Callers hold prepost_mutex() and use it stream-ordered.
void* prepost_scratch(int dev, size_t bytes);

}  // namespace gp
