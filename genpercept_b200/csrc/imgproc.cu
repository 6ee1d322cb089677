// Pre/post-processing around the hot path (SURVEY.md §8 row f1), on the GPU:
//   * separable anti-aliased bilinear / bicubic resize = torchvision.transforms.functional.resize(tensor,
//     antialias=True): uint8 -> float32 -> F.interpolate(antialias=True) -> torch.round -> uint8
//     (/root/reference/genpercept/util/image_util.py:75-105, genpercept_pipeline.py:301-307); the window /
//     weight arithmetic restates ATen's _compute_indices_min_size_weights_aa in float32
//   * colour-map lookup + 8-bit quantisation (image_util.py:25-63, genpercept_pipeline.py:318-321)
//   * uint8 / uint16 quantisation of the prediction (run.py:449-455)
// HBM-bound element-wise work: one thread per output element, coalesced along W; the weight tables
// (<= a few KB) are built on the host once per (in, out, mode) and cached on the device.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <map>
#include <mutex>
#include <stdexcept>
#include <string>
#include <tuple>
#include <vector>

#include "prepost.h"

namespace gp {
namespace {

struct AxisTable {          // device arrays
  int in_size = 0, out_size = 0, kmax = 0;
  int* xmin = nullptr;
  int* xsize = nullptr;
  float* w = nullptr;       // [out_size][kmax]
};

float aa_filter(float x, int mode) {
  x = fabsf(x);
  if (mode == 0) return x < 1.f ? 1.f - x : 0.f;
  const float a = -0.5f;    // ATen's anti-aliasing cubic
  if (x < 1.f) return ((a + 2.f) * x - (a + 3.f)) * x * x + 1.f;
  if (x < 2.f) return ((a * x - 5.f * a) * x + 8.f * a) * x - 4.f * a;
  return 0.f;
}

// float32 arithmetic in the order ATen uses (scale, support, center, window, normalisation by 1/total).
void build_axis(int in_size, int out_size, int mode, std::vector<int>& xmin, std::vector<int>& xsize, std::vector<float>& w,
                int* kmax_out) {
  const int interp = mode == 0 ? 2 : 4;
  const float scale = (float)in_size / (float)out_size;
  const float support = scale >= 1.f ? (interp * 0.5f) * scale : interp * 0.5f;
  const float invscale = scale >= 1.f ? 1.f / scale : 1.f;
  const int kmax = (int)ceilf(support) * 2 + 1;
  xmin.assign(out_size, 0);
  xsize.assign(out_size, 0);
  w.assign((size_t)out_size * kmax, 0.f);
  for (int i = 0; i < out_size; ++i) {
    const float center = scale * (float)(i + 0.5);
    int lo = (int)(center - support + 0.5f);
    if (lo < 0) lo = 0;
    int hi = (int)(center + support + 0.5f);
    if (hi > in_size) hi = in_size;
    int n = hi - lo;
    if (n < 0) n = 0;
    if (n > kmax) n = kmax;
    float tot = 0.f;
    float* wi = &w[(size_t)i * kmax];
    for (int j = 0; j < n; ++j) {
      wi[j] = aa_filter(((float)j + (float)lo - center + 0.5f) * invscale, mode);
      tot += wi[j];
    }
    if (tot != 0.f) {
      const float inv = 1.f / tot;
      for (int j = 0; j < n; ++j) wi[j] *= inv;
    }
    xmin[i] = lo;
    xsize[i] = n;
  }
  *kmax_out = kmax;
}

std::map<std::tuple<int, int, int, int>, AxisTable> g_tables;     // (device, in, out, mode)
struct Scratch { void* p = nullptr; size_t bytes = 0; };
std::map<int, Scratch> g_scratch;                                   // per device, grows

void ck(cudaError_t e, const char* what) { prepost_ck(e, what); }

const AxisTable& axis_table(int dev, int in_size, int out_size, int mode) {
  auto key = std::make_tuple(dev, in_size, out_size, mode);
  auto it = g_tables.find(key);
  if (it != g_tables.end()) return it->second;
  if (g_tables.size() >= 64) {   // every distinct (in, out) extent is a table: bound the cache (a folder of in-the-wild images)
    ck(cudaDeviceSynchronize(), "cudaDeviceSynchronize");
    for (auto& kv : g_tables) { cudaFree(kv.second.xmin); cudaFree(kv.second.xsize); cudaFree(kv.second.w); }
    g_tables.clear();
  }
  std::vector<int> xmin, xsize;
  std::vector<float> w;
  AxisTable t;
  t.in_size = in_size;
  t.out_size = out_size;
  build_axis(in_size, out_size, mode, xmin, xsize, w, &t.kmax);
  ck(cudaMalloc(reinterpret_cast<void**>(&t.xmin), xmin.size() * 4), "cudaMalloc");
  ck(cudaMalloc(reinterpret_cast<void**>(&t.xsize), xsize.size() * 4), "cudaMalloc");
  ck(cudaMalloc(reinterpret_cast<void**>(&t.w), w.size() * 4), "cudaMalloc");
  ck(cudaMemcpy(t.xmin, xmin.data(), xmin.size() * 4, cudaMemcpyHostToDevice), "cudaMemcpy");
  ck(cudaMemcpy(t.xsize, xsize.data(), xsize.size() * 4, cudaMemcpyHostToDevice), "cudaMemcpy");
  ck(cudaMemcpy(t.w, w.data(), w.size() * 4, cudaMemcpyHostToDevice), "cudaMemcpy");
  return g_tables.emplace(key, t).first->second;
}

__device__ __forceinline__ float ldf(const uint8_t* p, long long i) { return (float)p[i]; }
__device__ __forceinline__ float ldf(const float* p, long long i) { return p[i]; }

// width pass: src [N*H, W] -> dst f32 [N*H, OW]
template <typename TIn>
__global__ void aa_pass_w(const TIn* __restrict__ src, float* __restrict__ dst, long long rows, int W, int OW,
                          const int* __restrict__ xmin, const int* __restrict__ xsize, const float* __restrict__ w, int kmax) {
  const long long total = rows * OW;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ox = (int)(i % OW);
    const long long r = i / OW;
    const int lo = xmin[ox], n = xsize[ox];
    const float* wi = w + (size_t)ox * kmax;
    const long long base = r * W + lo;
    float acc = n > 0 ? ldf(src, base) * wi[0] : 0.f;
    for (int j = 1; j < n; ++j) acc = fmaf(ldf(src, base + j), wi[j], acc);
    dst[i] = acc;
  }
}

__device__ __forceinline__ void st_out(float* p, long long i, float v, int) { p[i] = v; }
__device__ __forceinline__ void st_out(uint8_t* p, long long i, float v, int clamp) {
  if (clamp) v = fminf(fmaxf(v, 0.f), 255.f);
  p[i] = (uint8_t)__float2int_rn(v);          // round half to even, like torch.round
}

// height pass: src f32 [N, H, OW] -> dst [N, OH, OW]
template <typename TOut>
__global__ void aa_pass_h(const float* __restrict__ src, TOut* __restrict__ dst, int N, int H, int OH, int OW,
                          const int* __restrict__ ymin, const int* __restrict__ ysize, const float* __restrict__ w, int kmax,
                          int clamp) {
  const long long total = (long long)N * OH * OW;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ox = (int)(i % OW);
    const long long t = i / OW;
    const int oy = (int)(t % OH);
    const long long n = t / OH;
    const int lo = ymin[oy], cnt = ysize[oy];
    const float* wi = w + (size_t)oy * kmax;
    const float* s = src + (n * H + lo) * OW + ox;
    float acc = cnt > 0 ? s[0] * wi[0] : 0.f;
    for (int j = 1; j < cnt; ++j) acc = fmaf(s[(long long)j * OW], wi[j], acc);
    st_out(dst, i, acc, clamp);
  }
}

template <typename TIn>
__global__ void cast_copy(const TIn* __restrict__ src, float* __restrict__ dst, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    dst[i] = ldf(src, i);
}

__global__ void colorize_kernel(const float* __restrict__ pred, uint8_t* __restrict__ out, long long n, float vmin,
                                float inv_range_den, const uint8_t* __restrict__ lut) {
  __shared__ uint8_t sl[768];
  for (int i = threadIdx.x; i < 768; i += blockDim.x) sl[i] = lut[i];
  __syncthreads();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float d = (pred[i] - vmin) / inv_range_den;          // (x - min) / (max - min), as image_util.py:45
    d = fminf(fmaxf(d, 0.f), 1.f);
    int idx = (int)(d * 256.f);
    idx = idx > 255 ? 255 : idx;
    out[3 * i + 0] = sl[3 * idx + 0];
    out[3 * i + 1] = sl[3 * idx + 1];
    out[3 * i + 2] = sl[3 * idx + 2];
  }
}

__global__ void quantize_kernel(const float* __restrict__ pred, void* __restrict__ out, long long n, int bits) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    if (bits == 16) reinterpret_cast<uint16_t*>(out)[i] = (uint16_t)(int)(pred[i] * 65535.0f);   // astype: truncation
    else reinterpret_cast<uint8_t*>(out)[i] = (uint8_t)(int)(pred[i] * 255.0f);
  }
}

int grid_for(long long n, int dev) {
  int sms = 132;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  long long b = (n + 255) / 256;
  const long long cap = (long long)sms * 8;               // a multiple of the SM count; grid-stride loops cover the rest
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

size_t esize(int dtype) { return dtype == GP_U8 ? 1 : 4; }

}  // namespace

std::mutex& prepost_mutex() {
  static std::mutex mu;
  return mu;
}

void* prepost_scratch(int dev, size_t bytes) {
  Scratch& s = g_scratch[dev];
  if (s.bytes < bytes) {
    if (s.p) ck(cudaFree(s.p), "cudaFree");
    s.p = nullptr;
    s.bytes = 0;
    ck(cudaMalloc(&s.p, bytes), "cudaMalloc");
    s.bytes = bytes;
  }
  return s.p;
}

}  // namespace gp

using namespace gp;

extern "C" {

gp_status gp_resize_aa(const void* src, int src_dtype, int src_on_host, int N, int H, int W, void* dst, int dst_dtype,
                       int dst_on_host, int OH, int OW, int mode, void* stream) {
  return prepost_guarded([&]() {
    if (!src || !dst || N < 1 || H < 1 || W < 1 || OH < 1 || OW < 1 || (mode != 0 && mode != 1) ||
        (src_dtype != GP_U8 && src_dtype != GP_F32) || (dst_dtype != GP_U8 && dst_dtype != GP_F32))
      throw std::invalid_argument("gp_resize_aa: bad arguments");
    std::lock_guard<std::mutex> lock(prepost_mutex());
    int dev = 0;
    ck(cudaGetDevice(&dev), "cudaGetDevice (no CUDA device: this library has no CPU path)");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const size_t n_in = (size_t)N * H * W, n_mid = (size_t)N * H * OW, n_out = (size_t)N * OH * OW;
    // scratch layout: [staged input][width-pass result f32][staged output]
    const size_t in_b = src_on_host ? (n_in * esize(src_dtype) + 255) / 256 * 256 : 0;
    const size_t mid_b = (n_mid * 4 + 255) / 256 * 256;
    const size_t out_b = dst_on_host ? (n_out * esize(dst_dtype) + 255) / 256 * 256 : 0;
    uint8_t* sc = static_cast<uint8_t*>(prepost_scratch(dev, in_b + mid_b + out_b));
    const void* d_src = src;
    if (src_on_host) {
      ck(cudaMemcpyAsync(sc, src, n_in * esize(src_dtype), cudaMemcpyHostToDevice, s), "H2D");
      d_src = sc;
    }
    float* mid = reinterpret_cast<float*>(sc + in_b);
    void* d_dst = dst_on_host ? static_cast<void*>(sc + in_b + mid_b) : dst;
    // width pass (or a cast when the width is unchanged)
    if (W != OW) {
      const AxisTable& tw = axis_table(dev, W, OW, mode);
      const int g = grid_for((long long)n_mid, dev);
      if (src_dtype == GP_U8)
        aa_pass_w<uint8_t><<<g, 256, 0, s>>>(static_cast<const uint8_t*>(d_src), mid, (long long)N * H, W, OW, tw.xmin, tw.xsize, tw.w, tw.kmax);
      else
        aa_pass_w<float><<<g, 256, 0, s>>>(static_cast<const float*>(d_src), mid, (long long)N * H, W, OW, tw.xmin, tw.xsize, tw.w, tw.kmax);
    } else {
      const int g = grid_for((long long)n_mid, dev);
      if (src_dtype == GP_U8) cast_copy<uint8_t><<<g, 256, 0, s>>>(static_cast<const uint8_t*>(d_src), mid, (long long)n_mid);
      else cast_copy<float><<<g, 256, 0, s>>>(static_cast<const float*>(d_src), mid, (long long)n_mid);
    }
    ck(cudaGetLastError(), "aa width pass");
    // height pass (identity table when the height is unchanged: window of one tap, weight 1)
    const AxisTable& th = axis_table(dev, H, OH, H == OH ? 0 : mode);
    const int g = grid_for((long long)n_out, dev);
    const int clamp = mode == 1 ? 1 : 0;                   // torchvision clamps only the bicubic result
    if (dst_dtype == GP_U8)
      aa_pass_h<uint8_t><<<g, 256, 0, s>>>(mid, static_cast<uint8_t*>(d_dst), N, H, OH, OW, th.xmin, th.xsize, th.w, th.kmax, clamp);
    else
      aa_pass_h<float><<<g, 256, 0, s>>>(mid, static_cast<float*>(d_dst), N, H, OH, OW, th.xmin, th.xsize, th.w, th.kmax, 0);
    ck(cudaGetLastError(), "aa height pass");
    if (dst_on_host) ck(cudaMemcpyAsync(dst, d_dst, n_out * esize(dst_dtype), cudaMemcpyDeviceToHost, s), "D2H");
    if (src_on_host || dst_on_host) ck(cudaStreamSynchronize(s), "sync");
  });
}

gp_status gp_colorize(const float* pred, int pred_on_host, int B, int H, int W, float vmin, float vmax,
                      const uint8_t* lut768_host, uint8_t* out_hwc, int out_on_host, void* stream) {
  return prepost_guarded([&]() {
    if (!pred || !lut768_host || !out_hwc || B < 1 || H < 1 || W < 1 || !(vmax > vmin))
      throw std::invalid_argument("gp_colorize: bad arguments");
    std::lock_guard<std::mutex> lock(prepost_mutex());
    int dev = 0;
    ck(cudaGetDevice(&dev), "cudaGetDevice (no CUDA device: this library has no CPU path)");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const size_t n = (size_t)B * H * W;
    const size_t in_b = pred_on_host ? (n * 4 + 255) / 256 * 256 : 0;
    const size_t out_b = out_on_host ? (n * 3 + 255) / 256 * 256 : 0;
    uint8_t* sc = static_cast<uint8_t*>(prepost_scratch(dev, 1024 + in_b + out_b));
    ck(cudaMemcpyAsync(sc, lut768_host, 768, cudaMemcpyHostToDevice, s), "lut H2D");
    const float* d_pred = pred;
    if (pred_on_host) {
      ck(cudaMemcpyAsync(sc + 1024, pred, n * 4, cudaMemcpyHostToDevice, s), "H2D");
      d_pred = reinterpret_cast<const float*>(sc + 1024);
    }
    uint8_t* d_out = out_on_host ? sc + 1024 + in_b : out_hwc;
    colorize_kernel<<<grid_for((long long)n, dev), 256, 0, s>>>(d_pred, d_out, (long long)n, vmin, vmax - vmin, sc);
    ck(cudaGetLastError(), "colorize");
    if (out_on_host) ck(cudaMemcpyAsync(out_hwc, d_out, n * 3, cudaMemcpyDeviceToHost, s), "D2H");
    ck(cudaStreamSynchronize(s), "sync");                  // the host LUT buffer may be released by the caller
  });
}

gp_status gp_quantize(const float* pred, int pred_on_host, size_t n, int bits, void* out, int out_on_host, void* stream) {
  return prepost_guarded([&]() {
    if (!pred || !out || n < 1 || (bits != 8 && bits != 16)) throw std::invalid_argument("gp_quantize: bad arguments");
    std::lock_guard<std::mutex> lock(prepost_mutex());
    int dev = 0;
    ck(cudaGetDevice(&dev), "cudaGetDevice (no CUDA device: this library has no CPU path)");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const size_t ob = bits / 8;
    const size_t in_b = pred_on_host ? (n * 4 + 255) / 256 * 256 : 0;
    const size_t out_b = out_on_host ? (n * ob + 255) / 256 * 256 : 0;
    uint8_t* sc = (in_b + out_b) ? static_cast<uint8_t*>(prepost_scratch(dev, in_b + out_b)) : nullptr;
    const float* d_pred = pred;
    if (pred_on_host) {
      ck(cudaMemcpyAsync(sc, pred, n * 4, cudaMemcpyHostToDevice, s), "H2D");
      d_pred = reinterpret_cast<const float*>(sc);
    }
    void* d_out = out_on_host ? static_cast<void*>(sc + in_b) : out;
    quantize_kernel<<<grid_for((long long)n, dev), 256, 0, s>>>(d_pred, d_out, (long long)n, bits);
    ck(cudaGetLastError(), "quantize");
    if (out_on_host) ck(cudaMemcpyAsync(out, d_out, n * ob, cudaMemcpyDeviceToHost, s), "D2H");
    if (pred_on_host || out_on_host) ck(cudaStreamSynchronize(s), "sync");
  });
}

}  // extern "C"
