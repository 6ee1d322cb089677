// Depth evaluation on the GPU (SURVEY.md §8 f4): the least-squares alignment of the reference's eval.py and its ten
// metrics, as two bandwidth-bound passes over B maps of H x W (pred fp32, gt fp32, valid uint8):
//   * alignment statistics: per image n, Σp, Σp², Σg, Σpg (fp64) and min / max p over the valid pixels of the grid
//     align_depth_least_square fits, then one block per image solves the 2 x 2 system as np.linalg.lstsq does;
//   * metrics: per pixel the alignment, the disparity -> depth conversion and the dataset clips in fp32 (the reference's
//     numpy float32 rounding), then per image the sums of the ten metrics of eval.py (fp64), finished by one block per
//     image.
// Each block writes fp64 partials; the per-image step reduces them in a fixed order, so there are no atomics and the
// results are bit-identical run to run.  The partials live in the pre/post scratch buffer (prepost.h).
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "launch.h"
#include "prepost.h"
#include "status.h"

namespace gp {
namespace {

constexpr int kThreads = 256;
constexpr int kAlignSlots = 7;     // n, Σp, Σp², Σg, Σpg, min p, max p
constexpr int kMetricSlots = 11;   // n, Σ|d|/g, Σd²/g, Σd², Σℓ², Σℓ, Σ|Δlog10|, #δ1, #δ2, #δ3, Σ(1/p - 1/g)²  (d = p - g, ℓ = ln p - ln g)
constexpr int kMetrics = 10;

// torch.nn.Upsample(scale_factor=s, mode="nearest"): source index of output index `dst` (ATen's nearest_idx with the
// user's scale: float(1/s), a float product, floorf, clamped to the last input index).
__device__ __forceinline__ int nearest_src(int dst, float inv_scale, int in_size) {
  const int s = (int)floorf(__fmul_rn((float)dst, inv_scale));
  return s < in_size - 1 ? s : in_size - 1;
}

// Calls f(p, g, valid) for every pixel of one image in grid-stride order: 128-bit loads of pred / gt (32-bit of the
// mask) where all three are aligned, a scalar loop for the tail or otherwise.  valid == nullptr: every pixel is valid.
template <typename F>
__device__ __forceinline__ void for_each_pixel(const float* __restrict__ P, const float* __restrict__ G,
                                               const uint8_t* __restrict__ V, long long n, F&& f) {
  const long long tid = (long long)blockIdx.x * kThreads + threadIdx.x;
  const long long stride = (long long)gridDim.x * kThreads;
  long long head = 0;
  if ((((uintptr_t)P | (uintptr_t)G) & 15) == 0 && ((uintptr_t)V & 3) == 0) {
    const long long nq = n >> 2;
    for (long long q = tid; q < nq; q += stride) {
      const float4 p = __ldg(reinterpret_cast<const float4*>(P) + q);
      const float4 g = __ldg(reinterpret_cast<const float4*>(G) + q);
      const uchar4 m = V ? __ldg(reinterpret_cast<const uchar4*>(V) + q) : make_uchar4(1, 1, 1, 1);
      f(p.x, g.x, m.x != 0);
      f(p.y, g.y, m.y != 0);
      f(p.z, g.z, m.z != 0);
      f(p.w, g.w, m.w != 0);
    }
    head = nq << 2;
  }
  for (long long i = head + tid; i < n; i += stride) f(__ldg(P + i), __ldg(G + i), V ? __ldg(V + i) != 0 : true);
}

// Fixed-order block reduction of N per-thread values (a shuffle tree per warp, then warp 0's lanes in order); slot k
// combines with op(k, a, b).  The result is valid in thread 0.
template <int N, typename Op>
__device__ __forceinline__ void block_reduce(double (&v)[N], Op op) {
  __shared__ double sm[kThreads / 32][N];
  for (int k = 0; k < N; ++k)
    for (int o = 16; o > 0; o >>= 1) v[k] = op(k, v[k], __shfl_down_sync(0xffffffffu, v[k], o));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0)
    for (int k = 0; k < N; ++k) sm[warp][k] = v[k];
  __syncthreads();
  if (threadIdx.x == 0)
    for (int k = 0; k < N; ++k) {
      double acc = sm[0][k];
      for (int w = 1; w < kThreads / 32; ++w) acc = op(k, acc, sm[w][k]);
      v[k] = acc;
    }
}

struct AlignOp {
  __device__ double operator()(int k, double a, double b) const { return k == 5 ? fmin(a, b) : k == 6 ? fmax(a, b) : a + b; }
};
struct SumOp {
  __device__ double operator()(int, double a, double b) const { return a + b; }
};

// mode 0: fit gt as given; mode 1 (least_square_disparity): the target is 1/g where g > 0 and the mask also needs
// g > 0 and p > 0 (eval.py:177-197).  fit_w < W: the fit reads the nearest-downscaled grid (H x fit_w; the reference's
// Upsample sees [1, H, W] as a 1-D signal of W samples over H channels, so only the width shrinks).
__global__ void __launch_bounds__(kThreads) align_stats_kernel(const float* __restrict__ pred, const float* __restrict__ gt,
                                                               const uint8_t* __restrict__ valid, int H, int W, int mode,
                                                               int fit_w, float inv_scale, double* __restrict__ partials) {
  const long long npix = (long long)H * W;
  const float* P = pred + blockIdx.y * npix;
  const float* G = gt + blockIdx.y * npix;
  const uint8_t* V = valid ? valid + blockIdx.y * npix : nullptr;
  double n = 0, sp = 0, spp = 0, sg = 0, spg = 0;
  float lo = INFINITY, hi = -INFINITY;
  auto px = [&](float p, float g, bool m) {
    if (mode == 1) {
      m = m && g > 0.f && p > 0.f;
      g = g > 0.f ? __frcp_rn(g) : 0.f;
    }
    if (!m) return;
    const double pd = p, gd = g;     // fp32 products are exact in fp64
    n += 1.0;
    sp += pd;
    spp += pd * pd;
    sg += gd;
    spg += pd * gd;
    lo = fminf(lo, p);
    hi = fmaxf(hi, p);
  };
  if (fit_w == W) {
    for_each_pixel(P, G, V, npix, px);
  } else {
    const long long nfit = (long long)H * fit_w;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < nfit; i += (long long)gridDim.x * kThreads) {
      const long long y = i / fit_w;
      const long long src = y * W + nearest_src((int)(i - y * fit_w), inv_scale, W);
      px(__ldg(P + src), __ldg(G + src), V ? __ldg(V + src) != 0 : true);
    }
  }
  double v[kAlignSlots] = {n, sp, spp, sg, spg, (double)lo, (double)hi};
  block_reduce(v, AlignOp());
  if (threadIdx.x == 0) {
    double* out = partials + ((long long)blockIdx.y * gridDim.x + blockIdx.x) * kAlignSlots;
    for (int k = 0; k < kAlignSlots; ++k) out[k] = v[k];
  }
}

// One block per image: reduce the partials in a fixed order, then the solution np.linalg.lstsq returns for
// A = [p 1], b = g, rounded to float32 (the dtype lstsq returns for float32 inputs):
//   n == 0            -> (0, 0)  (the empty system)
//   all p equal (= c) -> the minimum-norm solution of the rank-1 system, (c, 1) * Σg / (n (c² + 1))
//   otherwise         -> the normal equations in centred form.
__global__ void __launch_bounds__(kThreads) align_solve_kernel(const double* __restrict__ partials, int nblk,
                                                               float* __restrict__ scale_shift) {
  double v[kAlignSlots] = {0, 0, 0, 0, 0, INFINITY, -INFINITY};
  const double* p = partials + (long long)blockIdx.x * nblk * kAlignSlots;
  AlignOp op;
  for (int j = threadIdx.x; j < nblk; j += kThreads)
    for (int k = 0; k < kAlignSlots; ++k) v[k] = op(k, v[k], p[(long long)j * kAlignSlots + k]);
  block_reduce(v, op);
  if (threadIdx.x != 0) return;
  const double n = v[0], sp = v[1], spp = v[2], sg = v[3], spg = v[4];
  double scale = 0.0, shift = 0.0;
  if (n > 0.0) {
    if (v[5] == v[6]) {
      const double c = v[5], den = n * (c * c + 1.0);
      scale = c * sg / den;
      shift = sg / den;
    } else {
      const double mp = sp / n, mg = sg / n;
      scale = (spg / n - mp * mg) / (spp / n - mp * mp);
      shift = mg - scale * mp;
    }
  }
  scale_shift[2 * blockIdx.x] = (float)scale;
  scale_shift[2 * blockIdx.x + 1] = (float)shift;
}

// align_depth_least_square's return value: pred * scale + shift in float32, no FMA contraction.
__global__ void __launch_bounds__(kThreads) apply_alignment_kernel(const float* __restrict__ pred,
                                                                   const float* __restrict__ scale_shift, long long npix,
                                                                   long long total, float* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
    const long long b = i / npix;
    out[i] = __fadd_rn(__fmul_rn(pred[i], scale_shift[2 * b]), scale_shift[2 * b + 1]);
  }
}

// mode 0: pred as given; 1: pred * scale + shift; 2: the same in disparity, clipped at 1e-3 and inverted.  Then the
// dataset clip [min_depth, max_depth] and the clip at 1e-6 (eval.py:199-205; NaN passes through like np.clip).  The
// per-pixel terms are the reference's float32 expressions; their sums are fp64.
__global__ void __launch_bounds__(kThreads) metrics_kernel(const float* __restrict__ pred, const float* __restrict__ gt,
                                                           const uint8_t* __restrict__ valid, long long npix, int mode,
                                                           const float* __restrict__ scale_shift, float min_depth,
                                                           float max_depth, double* __restrict__ partials) {
  const long long b = blockIdx.y;
  const float* P = pred + b * npix;
  const float* G = gt + b * npix;
  const uint8_t* V = valid ? valid + b * npix : nullptr;
  const float s = mode ? scale_shift[2 * b] : 1.f, t = mode ? scale_shift[2 * b + 1] : 0.f;
  double v[kMetricSlots] = {};
  auto px = [&](float p, float g, bool m) {
    if (!m) return;
    if (mode) {
      p = __fadd_rn(__fmul_rn(p, s), t);
      if (mode == 2) {
        p = p < 1e-3f ? 1e-3f : p;
        p = __frcp_rn(p);
      }
    }
    p = p < min_depth ? min_depth : p;
    p = p > max_depth ? max_depth : p;
    p = p < 1e-6f ? 1e-6f : p;
    const float d = __fsub_rn(p, g), ad = fabsf(d);
    const float l = __fsub_rn(logf(p), logf(g));
    const float r = fmaxf(__fdiv_rn(p, g), __fdiv_rn(g, p));
    const float iv = __fsub_rn(__frcp_rn(p), __frcp_rn(g));
    v[0] += 1.0;
    v[1] += (double)__fdiv_rn(ad, g);
    v[2] += (double)__fdiv_rn(__fmul_rn(ad, ad), g);
    v[3] += (double)__fmul_rn(d, d);
    v[4] += (double)__fmul_rn(l, l);
    v[5] += (double)l;
    v[6] += (double)fabsf(__fsub_rn(log10f(p), log10f(g)));
    v[7] += r < 1.25f ? 1.0 : 0.0;
    v[8] += r < 1.5625f ? 1.0 : 0.0;
    v[9] += r < 1.953125f ? 1.0 : 0.0;
    v[10] += (double)__fmul_rn(iv, iv);
  };
  for_each_pixel(P, G, V, npix, px);
  block_reduce(v, SumOp());
  if (threadIdx.x == 0) {
    double* out = partials + (b * gridDim.x + blockIdx.x) * kMetricSlots;
    for (int k = 0; k < kMetricSlots; ++k) out[k] = v[k];
  }
}

// One block per image: fixed-order reduction, then the ten values in eval.py's order (eval.py:42-53).
__global__ void __launch_bounds__(kThreads) metrics_finish_kernel(const double* __restrict__ partials, int nblk,
                                                                  double* __restrict__ metrics) {
  double v[kMetricSlots] = {};
  const double* p = partials + (long long)blockIdx.x * nblk * kMetricSlots;
  for (int j = threadIdx.x; j < nblk; j += kThreads)
    for (int k = 0; k < kMetricSlots; ++k) v[k] += p[(long long)j * kMetricSlots + k];
  block_reduce(v, SumOp());
  if (threadIdx.x != 0) return;
  const double n = v[0], mean_l = v[5] / n;
  double* m = metrics + (long long)blockIdx.x * kMetrics;
  m[0] = v[1] / n;                                   // abs_relative_difference
  m[1] = v[2] / n;                                   // squared_relative_difference
  m[2] = sqrt(v[3] / n);                             // rmse_linear
  m[3] = sqrt(v[4] / n);                             // rmse_log
  m[4] = v[6] / n;                                   // log10
  m[5] = v[7] / n;                                   // delta1_acc
  m[6] = v[8] / n;                                   // delta2_acc
  m[7] = v[9] / n;                                   // delta3_acc
  m[8] = sqrt(v[10] / n);                            // i_rmse
  m[9] = sqrt(v[4] / n - mean_l * mean_l) * 100.0;   // silog_rmse
}

// Blocks per image: about four pixels per thread, at most ~8 blocks per SM over the whole batch.
int blocks_per_image(long long work, int B) {
  int dev = 0, sms = 132;
  GP_CUDA(cudaGetDevice(&dev));
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const long long want = (work + kThreads * 4 - 1) / (kThreads * 4);
  const long long cap = ((long long)sms * 8 + B - 1) / B;
  return (int)(want < 1 ? 1 : (want > cap ? cap : want));
}

void check_shape(const char* fn, const void* pred, const void* gt, int B, int H, int W) {
  GP_REQUIRE(pred && gt && B >= 1 && B <= 65535 && H >= 1 && W >= 1, std::string(fn) + ": bad arguments");
}

}  // namespace
}  // namespace gp

using namespace gp;

extern "C" {

gp_status gp_depth_align(const float* pred, const float* gt, const uint8_t* valid, int B, int H, int W, int mode,
                         int max_res, float* scale_shift_out, float* aligned_out, void* stream) {
  return guarded_call([&]() {
    check_shape("gp_depth_align", pred, gt, B, H, W);
    GP_REQUIRE(scale_shift_out && (mode == 0 || mode == 1) && max_res >= 0, "gp_depth_align: bad arguments");
    // align_depth_least_square (alignment.py:43-53): s = min(max_res / (H, W)) in fp64; below 1 the fit grid is
    // H x floor(W * s) (the output size torch computes for a 1-D nearest upsample).
    int fit_w = W;
    float inv_scale = 1.f;
    if (max_res > 0) {
      const double s = fmin((double)max_res / H, (double)max_res / W);
      if (s < 1.0) {
        fit_w = (int)floor((double)W * s);
        inv_scale = (float)(1.0 / s);
      }
    }
    GP_REQUIRE(fit_w >= 1, "gp_depth_align: max_res leaves an empty fit grid");
    std::lock_guard<std::mutex> lock(prepost_mutex());
    int dev = 0;
    GP_CUDA(cudaGetDevice(&dev));
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const int nblk = blocks_per_image((long long)H * fit_w, B);
    double* partials = static_cast<double*>(prepost_scratch(dev, (size_t)B * nblk * kAlignSlots * sizeof(double)));
    GP_CUDA(launch(align_stats_kernel, dim3(nblk, B), dim3(kThreads), 0, s, pred, gt, valid, H, W, mode, fit_w, inv_scale,
                   partials));
    GP_CUDA(launch(align_solve_kernel, dim3(B), dim3(kThreads), 0, s, partials, nblk, scale_shift_out));
    if (aligned_out) {
      const long long npix = (long long)H * W, total = npix * B;
      const int g = blocks_per_image(total, 1);
      GP_CUDA(launch(apply_alignment_kernel, dim3(g), dim3(kThreads), 0, s, pred, scale_shift_out, npix, total,
                     aligned_out));
    }
  });
}

gp_status gp_depth_metrics(const float* pred, const float* gt, const uint8_t* valid, int B, int H, int W, int mode,
                           const float* scale_shift, float min_depth, float max_depth, double* metrics_out, void* stream) {
  return guarded_call([&]() {
    check_shape("gp_depth_metrics", pred, gt, B, H, W);
    GP_REQUIRE(metrics_out && mode >= 0 && mode <= 2 && (mode == 0 || scale_shift), "gp_depth_metrics: bad arguments");
    std::lock_guard<std::mutex> lock(prepost_mutex());
    int dev = 0;
    GP_CUDA(cudaGetDevice(&dev));
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const long long npix = (long long)H * W;
    const int nblk = blocks_per_image(npix, B);
    double* partials = static_cast<double*>(prepost_scratch(dev, (size_t)B * nblk * kMetricSlots * sizeof(double)));
    GP_CUDA(launch(metrics_kernel, dim3(nblk, B), dim3(kThreads), 0, s, pred, gt, valid, npix, mode, scale_shift,
                   min_depth, max_depth, partials));
    GP_CUDA(launch(metrics_finish_kernel, dim3(B), dim3(kThreads), 0, s, partials, nblk, metrics_out));
  });
}

}  // extern "C"
