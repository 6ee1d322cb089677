// Pre/post-processing around the hot path (SURVEY.md §8 row f1), on the GPU:
//   * separable anti-aliased bilinear / bicubic resize = torchvision.transforms.functional.resize(tensor,
//     antialias=True): uint8 -> float32 -> F.interpolate(antialias=True) -> torch.round -> uint8
//     (/root/reference/genpercept/util/image_util.py:75-105, genpercept_pipeline.py:301-307); the window /
//     weight arithmetic restates ATen's _compute_indices_min_size_weights_aa in float32
//   * colour-map lookup + 8-bit quantisation (image_util.py:25-63, genpercept_pipeline.py:318-321)
//   * uint8 / uint16 quantisation of the prediction (run.py:449-455)
//   * GenPercept v1 (GenPercept_v1/genpercept/pipeline_genpercept.py): PIL.Image.resize(size) with its default BICUBIC
//     filter, byte for byte (Pillow's Resample.c: double coefficients normalised per window and rounded to 22-bit fixed
//     point, int32 passes, the horizontal one over only the rows the vertical one reads), and the post-processing of
//     __call__ (F.interpolate back to the input size, per-image min-max depth, norm_to_rgb, the uint8 seg / sr map)
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
  int32_t* wq = nullptr;    // Pillow tables (mode 2): fixed-point coefficients [out_size][kmax], no float weights
  int first = 0, last = 0;  // Pillow tables: the input extent [first, last) the windows read
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

// Pillow's precompute_coeffs + normalize_coeffs_8bpc for the BICUBIC filter (a = -0.5, support 2), in double and in its
// order: window [xmin, xmin + n) around center = (i + 0.5) * scale, weights normalised by their sum, then rounded away
// from zero to 22 fractional bits.
double pil_bicubic(double x) {
  const double a = -0.5;
  if (x < 0.0) x = -x;
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
  if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
  return 0.0;
}

constexpr int kPilBits = 22;      // PRECISION_BITS = 32 - 8 - 2 for 8-bit images

void build_axis_pil(int in_size, int out_size, std::vector<int>& xmin, std::vector<int>& xsize, std::vector<int32_t>& wq,
                    int* kmax_out) {
  const double scale = (double)in_size / out_size;
  const double filterscale = scale < 1.0 ? 1.0 : scale;
  const double support = 2.0 * filterscale;
  const int kmax = (int)ceil(support) * 2 + 1;
  xmin.assign(out_size, 0);
  xsize.assign(out_size, 0);
  wq.assign((size_t)out_size * kmax, 0);
  std::vector<double> k(kmax);
  for (int i = 0; i < out_size; ++i) {
    const double center = (i + 0.5) * scale;
    const double ss = 1.0 / filterscale;
    int lo = (int)(center - support + 0.5);
    if (lo < 0) lo = 0;
    int hi = (int)(center + support + 0.5);
    if (hi > in_size) hi = in_size;
    const int n = hi - lo;
    double ww = 0.0;
    for (int j = 0; j < n; ++j) {
      k[j] = pil_bicubic((j + lo - center + 0.5) * ss);
      ww += k[j];
    }
    for (int j = 0; j < n; ++j) {
      const double v = ww != 0.0 ? k[j] / ww : k[j];
      wq[(size_t)i * kmax + j] = v < 0 ? (int32_t)(-0.5 + v * (1 << kPilBits)) : (int32_t)(0.5 + v * (1 << kPilBits));
    }
    xmin[i] = lo;
    xsize[i] = n;
  }
  *kmax_out = kmax;
}

std::map<std::tuple<int, int, int, int>, AxisTable> g_tables;     // (device, in, out, mode); mode 2 = Pillow's bicubic
struct Scratch { void* p = nullptr; size_t bytes = 0; };
std::map<int, Scratch> g_scratch;                                   // per device, grows

void ck(cudaError_t e, const char* what) { prepost_ck(e, what); }

const AxisTable& axis_table(int dev, int in_size, int out_size, int mode) {
  auto key = std::make_tuple(dev, in_size, out_size, mode);
  auto it = g_tables.find(key);
  if (it != g_tables.end()) return it->second;
  if (g_tables.size() >= 64) {   // every distinct (in, out) extent is a table: bound the cache (a folder of in-the-wild images)
    ck(cudaDeviceSynchronize(), "cudaDeviceSynchronize");
    for (auto& kv : g_tables) {
      cudaFree(kv.second.xmin);
      cudaFree(kv.second.xsize);
      cudaFree(kv.second.w);
      cudaFree(kv.second.wq);
    }
    g_tables.clear();
  }
  std::vector<int> xmin, xsize;
  std::vector<float> w;
  std::vector<int32_t> wq;
  AxisTable t;
  t.in_size = in_size;
  t.out_size = out_size;
  if (mode == 2) {
    build_axis_pil(in_size, out_size, xmin, xsize, wq, &t.kmax);
    t.first = xmin[0];
    t.last = xmin[out_size - 1] + xsize[out_size - 1];
  } else {
    build_axis(in_size, out_size, mode, xmin, xsize, w, &t.kmax);
  }
  ck(cudaMalloc(reinterpret_cast<void**>(&t.xmin), xmin.size() * 4), "cudaMalloc");
  ck(cudaMalloc(reinterpret_cast<void**>(&t.xsize), xsize.size() * 4), "cudaMalloc");
  ck(cudaMemcpy(t.xmin, xmin.data(), xmin.size() * 4, cudaMemcpyHostToDevice), "cudaMemcpy");
  ck(cudaMemcpy(t.xsize, xsize.data(), xsize.size() * 4, cudaMemcpyHostToDevice), "cudaMemcpy");
  if (mode == 2) {
    ck(cudaMalloc(reinterpret_cast<void**>(&t.wq), wq.size() * 4), "cudaMalloc");
    ck(cudaMemcpy(t.wq, wq.data(), wq.size() * 4, cudaMemcpyHostToDevice), "cudaMemcpy");
  } else {
    ck(cudaMalloc(reinterpret_cast<void**>(&t.w), w.size() * 4), "cudaMalloc");
    ck(cudaMemcpy(t.w, w.data(), w.size() * 4, cudaMemcpyHostToDevice), "cudaMemcpy");
  }
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

// ---- Pillow's BICUBIC resize of an 8-bit RGB image (ImagingResampleHorizontal_8bpc / _Vertical_8bpc)
__device__ __forceinline__ uint8_t pil_clip8(int v) {   // clip8: the sum's integer part, clamped to 0..255
  v >>= kPilBits;
  return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// horizontal pass: rows of src HWC [rows, W, 3] -> dst HWC [rows, OW, 3], each channel rounded and clipped to uint8
__global__ void pil_pass_h(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int rows, int W, int OW,
                           const int* __restrict__ xmin, const int* __restrict__ xsize, const int32_t* __restrict__ k,
                           int kmax) {
  const long long total = (long long)rows * OW;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ox = (int)(i % OW);
    const long long r = i / OW;
    const int lo = xmin[ox], n = xsize[ox];
    const int32_t* ki = k + (size_t)ox * kmax;
    const uint8_t* s = src + (r * W + lo) * 3;
    int s0 = 1 << (kPilBits - 1), s1 = s0, s2 = s0;
    for (int j = 0; j < n; ++j) {
      const int c = ki[j];
      s0 += s[3 * j + 0] * c;
      s1 += s[3 * j + 1] * c;
      s2 += s[3 * j + 2] * c;
    }
    dst[3 * i + 0] = pil_clip8(s0);
    dst[3 * i + 1] = pil_clip8(s1);
    dst[3 * i + 2] = pil_clip8(s2);
  }
}

// vertical pass: src HWC [rows, OW, 3] whose first row is input row `row0` -> dst CHW [3, OH, OW]
__global__ void pil_pass_v(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int OH, int OW, int row0,
                           const int* __restrict__ ymin, const int* __restrict__ ysize, const int32_t* __restrict__ k,
                           int kmax) {
  const long long total = (long long)OH * OW;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ox = (int)(i % OW);
    const int oy = (int)(i / OW);
    const int lo = ymin[oy] - row0, n = ysize[oy];
    const int32_t* ki = k + (size_t)oy * kmax;
    const uint8_t* s = src + ((long long)lo * OW + ox) * 3;
    int s0 = 1 << (kPilBits - 1), s1 = s0, s2 = s0;
    for (int j = 0; j < n; ++j) {
      const int c = ki[j];
      const uint8_t* p = s + (long long)j * OW * 3;
      s0 += p[0] * c;
      s1 += p[1] * c;
      s2 += p[2] * c;
    }
    dst[i] = pil_clip8(s0);
    dst[total + i] = pil_clip8(s1);
    dst[2 * total + i] = pil_clip8(s2);
  }
}

// an unchanged height: the (possibly width-resampled) HWC rows as CHW planes
__global__ void hwc_to_chw(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, long long pixels) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < pixels; i += (long long)gridDim.x * blockDim.x) {
    dst[i] = src[3 * i + 0];
    dst[pixels + i] = src[3 * i + 1];
    dst[2 * pixels + i] = src[3 * i + 2];
  }
}

// ---- v1 post-processing: p = 2 y - 1 of the engine's map, then F.interpolate(size=(H, W)) in ATen's CUDA arithmetic
struct V1Interp {
  int h, w, H, W;
  float rh, rw;   // (float)in / out, area_pixel_compute_scale without scale factors
  int kind;       // 0 none (sizes equal, or match_input_res=False), 1 bilinear (align_corners=False), 2 nearest (legacy)
};

__device__ __forceinline__ float v1_p(const float* y, long long i) { return 2.f * y[i] - 1.f; }

__device__ __forceinline__ float v1_sample(const float* __restrict__ src, const V1Interp& g, int oy, int ox) {
  if (g.kind == 0) return v1_p(src, (long long)oy * g.w + ox);
  if (g.kind == 2) {                                   // nearest_neighbor_compute_source_index
    const int sy = min((int)floorf((float)oy * g.rh), g.h - 1);
    const int sx = min((int)floorf((float)ox * g.rw), g.w - 1);
    return v1_p(src, (long long)sy * g.w + sx);
  }
  float hr = g.rh * ((float)oy + 0.5f) - 0.5f;         // area_pixel_compute_source_index, clamped at 0
  if (hr < 0.f) hr = 0.f;
  float wr = g.rw * ((float)ox + 0.5f) - 0.5f;
  if (wr < 0.f) wr = 0.f;
  const int h1 = (int)hr, w1 = (int)wr;
  const int h1p = h1 < g.h - 1 ? 1 : 0, w1p = w1 < g.w - 1 ? 1 : 0;
  const float h1l = hr - (float)h1, h0l = 1.f - h1l;
  const float w1l = wr - (float)w1, w0l = 1.f - w1l;
  const float* r0 = src + (long long)h1 * g.w;
  const float* r1 = r0 + (long long)h1p * g.w;
  return h0l * (w0l * v1_p(r0, w1) + w1l * v1_p(r0, w1 + w1p)) + h1l * (w0l * v1_p(r1, w1) + w1l * v1_p(r1, w1 + w1p));
}

constexpr int kV1Threads = 256;

// depth, first pass: out[b] = interpolated p, and per block the (min, max) of its pixels -> partial[b][blockIdx.x]
__global__ void __launch_bounds__(kV1Threads) v1_depth_interp(const float* __restrict__ pred, float* __restrict__ out,
                                                              V1Interp g, float2* __restrict__ partial) {
  __shared__ float smn[kV1Threads], smx[kV1Threads];
  const int b = blockIdx.y;
  const long long n = (long long)g.H * g.W;
  const float* src = pred + (long long)b * g.h * g.w;
  float* dst = out + (long long)b * n;
  float mn = INFINITY, mx = -INFINITY;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = v1_sample(src, g, (int)(i / g.W), (int)(i % g.W));
    dst[i] = v;
    mn = fminf(mn, v);
    mx = fmaxf(mx, v);
  }
  smn[threadIdx.x] = mn;
  smx[threadIdx.x] = mx;
  __syncthreads();
  for (int o = kV1Threads / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      smn[threadIdx.x] = fminf(smn[threadIdx.x], smn[threadIdx.x + o]);
      smx[threadIdx.x] = fmaxf(smx[threadIdx.x], smx[threadIdx.x + o]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) partial[(long long)b * gridDim.x + blockIdx.x] = make_float2(smn[0], smx[0]);
}

// depth, second pass: every block reduces its image's partials in the same fixed order, then (x - min) / (max - min)
__global__ void __launch_bounds__(kV1Threads) v1_depth_normalise(float* __restrict__ out, long long n,
                                                                 const float2* __restrict__ partial, int nparts) {
  __shared__ float smn[kV1Threads], smx[kV1Threads];
  const int b = blockIdx.y;
  float mn = INFINITY, mx = -INFINITY;
  for (int j = threadIdx.x; j < nparts; j += kV1Threads) {
    const float2 p = partial[(long long)b * nparts + j];
    mn = fminf(mn, p.x);
    mx = fmaxf(mx, p.y);
  }
  smn[threadIdx.x] = mn;
  smx[threadIdx.x] = mx;
  __syncthreads();
  for (int o = kV1Threads / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      smn[threadIdx.x] = fminf(smn[threadIdx.x], smn[threadIdx.x + o]);
      smx[threadIdx.x] = fmaxf(smx[threadIdx.x], smx[threadIdx.x + o]);
    }
    __syncthreads();
  }
  const float lo = smn[0], den = smx[0] - smn[0];      // no clamp: a constant map gives 0 / 0 = NaN, as torch does
  float* dst = out + (long long)b * n;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    dst[i] = (dst[i] - lo) / den;
}

// normal: clip(p, -1, 1) -> out fp32 [B,3,H,W], and norm_to_rgb ((n + 1) * 0.5 * 255, clip, astype(uint8)) -> rgb [B,H,W,3]
__global__ void v1_normal(const float* __restrict__ pred, float* __restrict__ out, uint8_t* __restrict__ rgb, V1Interp g,
                          int B) {
  const long long hw = (long long)g.H * g.W, total = (long long)B * hw;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / hw, px = i % hw;
    const int oy = (int)(px / g.W), ox = (int)(px % g.W);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float v = v1_sample(pred + (b * 3 + c) * g.h * g.w, g, oy, ox);
      v = fminf(fmaxf(v, -1.f), 1.f);
      out[(b * 3 + c) * hw + px] = v;
      float t = ((v + 1.f) * 0.5f) * 255.f;
      t = fminf(fmaxf(t, 0.f), 255.f);
      rgb[3 * i + c] = (uint8_t)(int)t;
    }
  }
}

// seg / sr: ((p + 1) / 2 * 255).clip(0, 255).astype(uint8) -> out CHW [B,3,H,W]
__global__ void v1_seg(const float* __restrict__ pred, uint8_t* __restrict__ out, V1Interp g, int B) {
  const long long hw = (long long)g.H * g.W, total = (long long)B * 3 * hw;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long plane = i / hw, px = i % hw;
    const float v = v1_sample(pred + plane * g.h * g.w, g, (int)(px / g.W), (int)(px % g.W));
    float t = ((v + 1.f) / 2.f) * 255.f;
    t = fminf(fmaxf(t, 0.f), 255.f);
    out[i] = (uint8_t)(int)t;
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

gp_status gp_resize_pil(const uint8_t* src_hwc, int src_on_host, int H, int W, uint8_t* dst_chw, int dst_on_host, int OH,
                        int OW, void* stream) {
  return prepost_guarded([&]() {
    if (!src_hwc || !dst_chw || H < 1 || W < 1 || OH < 1 || OW < 1) throw std::invalid_argument("gp_resize_pil: bad arguments");
    std::lock_guard<std::mutex> lock(prepost_mutex());
    int dev = 0;
    ck(cudaGetDevice(&dev), "cudaGetDevice (no CUDA device: this library has no CPU path)");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    // the rows the vertical pass reads (Pillow: ybox_first .. ybox_last); all of them when the height is kept
    int row0 = 0, rows = H;
    if (H != OH) {
      const AxisTable& tv = axis_table(dev, H, OH, 2);
      row0 = tv.first;
      rows = tv.last - tv.first;
    }
    const size_t n_in = (size_t)H * W * 3, n_mid = (size_t)rows * OW * 3, n_out = (size_t)OH * OW * 3;
    // scratch layout: [staged input][horizontal-pass rows, uint8 HWC][staged output]
    const size_t in_b = src_on_host ? (n_in + 255) / 256 * 256 : 0;
    const size_t mid_b = W != OW ? (n_mid + 255) / 256 * 256 : 0;
    const size_t out_b = dst_on_host ? (n_out + 255) / 256 * 256 : 0;
    uint8_t* sc = (in_b + mid_b + out_b) ? static_cast<uint8_t*>(prepost_scratch(dev, in_b + mid_b + out_b)) : nullptr;
    const uint8_t* d_src = src_hwc;
    if (src_on_host) {
      ck(cudaMemcpyAsync(sc, src_hwc, n_in, cudaMemcpyHostToDevice, s), "H2D");
      d_src = sc;
    }
    uint8_t* d_dst = dst_on_host ? sc + in_b + mid_b : dst_chw;
    const uint8_t* cur = d_src + (size_t)row0 * W * 3;   // HWC rows [row0, row0 + rows) at width OW after this block
    if (W != OW) {
      const AxisTable& th = axis_table(dev, W, OW, 2);
      uint8_t* mid = sc + in_b;
      pil_pass_h<<<grid_for((long long)rows * OW, dev), 256, 0, s>>>(cur, mid, rows, W, OW, th.xmin, th.xsize, th.wq, th.kmax);
      ck(cudaGetLastError(), "pil horizontal pass");
      cur = mid;
    }
    if (H != OH) {   // looked up again: the width table's insertion may have evicted it (the cache is bounded)
      const AxisTable& tv = axis_table(dev, H, OH, 2);
      pil_pass_v<<<grid_for((long long)OH * OW, dev), 256, 0, s>>>(cur, d_dst, OH, OW, row0, tv.xmin, tv.xsize, tv.wq, tv.kmax);
      ck(cudaGetLastError(), "pil vertical pass");
    } else {
      hwc_to_chw<<<grid_for((long long)OH * OW, dev), 256, 0, s>>>(cur, d_dst, (long long)OH * OW);
      ck(cudaGetLastError(), "hwc_to_chw");
    }
    if (dst_on_host) ck(cudaMemcpyAsync(dst_chw, d_dst, n_out, cudaMemcpyDeviceToHost, s), "D2H");
    if (src_on_host || dst_on_host) ck(cudaStreamSynchronize(s), "sync");
  });
}

gp_status gp_v1_postprocess(const float* pred, int B, int C, int h, int w, int task, int H, int W, float* out_f32,
                            uint8_t* out_u8, void* stream) {
  return prepost_guarded([&]() {
    const bool ok = pred && B >= 1 && h >= 1 && w >= 1 && H >= 1 && W >= 1 &&
                    ((task == 0 && C == 1 && out_f32) || (task == 1 && C == 3 && out_f32 && out_u8) ||
                     (task == 2 && C == 3 && out_u8));
    if (!ok) throw std::invalid_argument("gp_v1_postprocess: bad arguments");
    std::lock_guard<std::mutex> lock(prepost_mutex());
    int dev = 0;
    ck(cudaGetDevice(&dev), "cudaGetDevice (no CUDA device: this library has no CPU path)");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    V1Interp g;
    g.h = h; g.w = w; g.H = H; g.W = W;
    g.rh = (float)h / (float)H;
    g.rw = (float)w / (float)W;
    g.kind = (H == h && W == w) ? 0 : (task == 2 ? 2 : 1);
    const long long n = (long long)H * W;
    if (task == 0) {
      long long parts = (n + 2047) / 2048;
      const int nparts = (int)(parts < 1 ? 1 : (parts > 256 ? 256 : parts));
      if (B > 65535) throw std::invalid_argument("gp_v1_postprocess: batch above 65535");
      float2* partial = static_cast<float2*>(prepost_scratch(dev, (size_t)B * nparts * sizeof(float2)));
      const dim3 grid(nparts, B);
      v1_depth_interp<<<grid, kV1Threads, 0, s>>>(pred, out_f32, g, partial);
      ck(cudaGetLastError(), "v1 depth interpolation");
      v1_depth_normalise<<<grid, kV1Threads, 0, s>>>(out_f32, n, partial, nparts);
      ck(cudaGetLastError(), "v1 depth normalisation");
    } else if (task == 1) {
      v1_normal<<<grid_for((long long)B * n, dev), 256, 0, s>>>(pred, out_f32, out_u8, g, B);
      ck(cudaGetLastError(), "v1 normal");
    } else {
      v1_seg<<<grid_for((long long)B * 3 * n, dev), 256, 0, s>>>(pred, out_u8, g, B);
      ck(cudaGetLastError(), "v1 seg");
    }
  });
}

}  // extern "C"
