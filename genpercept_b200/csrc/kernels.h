// Bandwidth-bound and small kernels of the hot path (everything that is not a dense contraction):
// GroupNorm(+SiLU), LayerNorm, row softmax, the 2-token cross-attention closed form,
// ReLU, bilinear 2x, direct convolution for tiny channel counts (and as the on-device triage
// reference for the wgmma kernels), pre/post-processing.  16-bit NHWC activations, fp32 math.
// `split` = the high-precision layout: C logical channels stored as [hi C | lo C] per pixel (two fp16 planes,
// value = hi + lo); rows of score matrices as [hi Tp | lo Tp].
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace gp {

enum DirectConvFlags : int {
  DC_RELU = 1,
  DC_OUT_F32_NCHW = 2,
  DC_UP2X = 8,          // input is nearest-2x upsampled before the convolution
};

struct DirectConvParams {
  const void* in;       // 16-bit NHWC, channel stride in_cstride
  int N, H, W, Cin, in_cstride;
  int in_lo, out_lo;    // high-precision layout: element offset of the lo plane inside a pixel (0 = plain 16-bit)
  const float* w;       // fp32 [ks*ks][Cin][Cout]
  const float* bias;    // fp32 [Cout] or null
  const void* res;      // 16-bit NHWC (out_cstride) or null
  void* out;
  int Ho, Wo, Cout, out_cstride;
  int ks, stride, pad;  // pad = leading zero padding (trailing padding is implicit)
  int flags;
};
cudaError_t direct_conv(const DirectConvParams& p, bool bf16, cudaStream_t s);

// GroupNorm, deterministic: per-chunk partials [N][chunks][Ctot][kGnRec] -> per-(n, channel)
// scale / shift -> apply.  chunks = gn_chunks(N, HW) for every source of one normalisation.
// A partial is (count, mean, M2) of one channel over its pixels, M2 = sum of squared deviations from that mean:
// the variance stays accurate at any mean / std ratio, where sum / sum-of-squares cancels.  A record of count 0
// (an untouched, zeroed slot) merges as nothing.
constexpr int kGnRec = 3;
int gn_chunks(int N, long long HW);
cudaError_t gn_stats(const void* x, int N, long long HW, int C, float* partial, int chunks, int Ctot, int coff,
                     bool bf16, cudaStream_t s, bool split = false);
// one source of a (possibly concatenated) normalisation: partials [N][chunks][C][kGnRec]; the partials
// come either from gn_stats or from the producing implicit-GEMM's epilogue (IgemmParams::stats).
struct GnSrc { const float* partial; int chunks; int C; };

#ifdef __CUDACC__
// Chan et al.'s pairwise update: (na, ma, m2a) <- the statistics of the union of a and (nb, mb, m2b).  The weight
// nb / n takes the fast division (2 ulp; an IEEE division is a called slow path, which costs the GEMM epilogue spills).
__device__ __forceinline__ void chan_merge(float& na, float& ma, float& m2a, float nb, float mb, float m2b) {
  const float n = na + nb;
  const float f = n > 0.f ? __fdividef(nb, n) : 0.f;
  const float d = mb - ma;
  ma = fmaf(d, f, ma);
  m2a = m2a + m2b + d * d * na * f;
  na = n;
}
#endif
cudaError_t gn_finalize(const GnSrc* srcs, int nsrc, const float* gamma, const float* beta, int N, int Ctot,
                        int groups, long long HW, float eps, float* scale_shift /*[N][Ctot][2]*/, cudaStream_t s);
cudaError_t gn_apply(const void* x, int N, long long HW, int C, const float* scale_shift, int Ctot,
                     int coff, void* y, int y_cstride, bool silu, bool bf16, cudaStream_t s, bool split = false);

cudaError_t layernorm(const void* x, void* y, long long tokens, int C, const float* gamma,
                      const float* beta, float eps, bool bf16, cudaStream_t s, bool split = false);
// in-place softmax over the first T entries of each row (row stride Tp elements).  Where T is a multiple of 8 (and
// >= 64) rows are limited to kSoftmaxRowsMaxT entries (cudaErrorInvalidValue beyond); other T have no limit.
constexpr int kSoftmaxRowsMaxT = 16384;
cudaError_t softmax_rows(void* s_inout, long long rows, int T, int Tp, bool bf16, cudaStream_t s, bool split = false);
// y = x + c0 + sigmoid(LN(x) . U + u0) . M     (SURVEY.md F6; U already carries LN gamma, u0 beta)
// Needs heads % 5 == 0, C % 32 == 0, C <= 1280 and U, M, c0, u0 within 226 KiB of shared memory (cudaErrorInvalidValue
// otherwise): the SD-2.1 UNet's 5 / 10 / 20 heads over C = 320 / 640 / 1280.
cudaError_t xattn2(const void* x, void* y, long long tokens, int C, int heads, const float* U /*[h][C]*/,
                   const float* u0 /*[h]*/, const float* M /*[h][C]*/, const float* c0 /*[C]*/,
                   float eps, bool bf16, cudaStream_t s, bool split = false);
// split_c: 0, or the logical channel count C of a high-precision [hi C | lo C] tensor (n = pixels * C)
cudaError_t relu16(const void* in, void* out, long long n, bool bf16, cudaStream_t s, int split_c = 0);
cudaError_t bilinear_up2x(const void* in, void* out, int N, int H, int W, int C, bool bf16,
                          cudaStream_t s, bool split = false);
// In-place softmax over each of `groups` consecutive runs of `n` columns of every row of x [rows, ld] (16-bit); columns
// beyond groups*n are left untouched (zero padding of the general cross-attention score matrix).
cudaError_t softmax_groups(void* x, long long rows, int ld, int groups, int n, bool bf16, cudaStream_t s, bool split = false);
// F.interpolate(size=(OH,OW), mode="nearest") on 16-bit NHWC: src = min(floor(dst * in/out), in-1)  (the UNet's
// Upsample2D with an explicit output size, when H/8 or W/8 is not a multiple of 8)
cudaError_t nearest_resize(const void* in, void* out, int N, int H, int W, int OH, int OW, int C, cudaStream_t s);
// F.interpolate(size=(OH,OW), mode="bilinear", align_corners=False) on 16-bit NHWC (the DPT fusion stage's resize of a
// skip feature to the running map's size, /root/reference/genpercept/models/dpt_head.py:297-300)
cudaError_t bilinear_resize(const void* in, void* out, int N, int H, int W, int OH, int OW, int C, bool bf16, cudaStream_t s,
                            bool split = false);
// latent I/O of encode_rgb / decode_pred: 16-bit NHWC8 <-> fp32 NCHW [N,4,H,W]; the second form applies
// y = M (x * pre) + b per pixel (post_quant_conv(latent / 0.18215), genpercept_pipeline.py:519-521)
cudaError_t nhwc8_to_nchw_f32(const void* in, float* out, int N, int H, int W, int c, bool bf16, cudaStream_t s, bool split = false);
cudaError_t nchw4_affine_to_nhwc8(const float* in, void* out, int N, int H, int W, float pre, const float* m /*[4][4] or null*/,
                                  const float* b /*[4] or null*/, bool bf16, cudaStream_t s, bool split = false);
// the high-precision latent's (hi, lo) pair without loss: split NHWC8 <-> fp32 NCHW [N,8,H,W] = [hi 0..3 | lo 0..3]
cudaError_t latent_pair_to_nchw(const void* in, float* out, int N, int H, int W, bool bf16, cudaStream_t s);
cudaError_t latent_pair_from_nchw(const float* in, void* out, int N, int H, int W, bool bf16, cudaStream_t s);
// u8 / f16 / f32 NCHW [N,3,H,W] (u8 is mapped x/255*2-1), K-packed for the VAE encoder's stem: 16-bit NHWC32 = the pixel's
// 3x3 neighbourhood along the channel axis [centre tap | 8 other taps row-major | 5 zeros]; im2col_tap_slot(r, q) gives a
// tap's position.
cudaError_t preprocess_rgb_im2col(const void* in, int in_kind /*0 u8, 1 f16, 2 f32*/, void* out, int N, int H, int W, bool bf16, cudaStream_t s,
                                  bool split = false);
inline int im2col_tap_slot(int r, int q) {      // 3x3 tap (r, q) -> group of 3 channels inside the NHWC32 pixel
  if (r == 1 && q == 1) return 0;
  const int lin = r * 3 + q;
  return lin < 4 ? lin + 1 : lin;
}
// Multi-step archs (SURVEY.md §8 f4), 16-bit NHWC8 latents: the UNet input of a step (in_ch 8: [rgb_latent | pred_latent],
// 4: pred_latent), the DDIM update (eta = 0; coefficients from genpercept_b200/scheduler.py, read from the device array
// c_dev[4]) and post_quant_conv(x / 0.18215).
cudaError_t latent_pack(const void* lat, const void* smp, void* xin, long long npx, int in_ch, bool bf16, cudaStream_t s, bool split = false);
cudaError_t ddim_step(const void* model_out, void* sample, void* x0, long long npx, const float* c_dev, bool bf16, cudaStream_t s,
                      bool split = false);
// One step's row of the multi-step bias table into the UNet's live conv1 bias buffers: segment k copies len floats from
// row + off to dst.  segs (device) holds nseg segments; one block per segment.
struct BiasSegment { float* dst; int off; int len; };
cudaError_t bias_scatter(const float* row, const BiasSegment* segs, int nseg, cudaStream_t s);
cudaError_t latent_affine(const void* in, void* out, long long npx, float pre, const float* mat, const float* bias, bool bf16,
                          cudaStream_t s, bool split = false);
// SD-2.1's CLIP text tower (text_tower, engine.cu), 16-bit or pair rows of tokens:
//   text_embed: out[t] = tok[ids[t]] + pos[t] (fp32 tables [*, C], the sum in fp32, then stored)
//   causal_attention: softmax(q k^T) v per head over keys j <= i, scores and softmax in fp32 (the scale folded into q);
//     qkv per token [q C | k C | v C] with C = heads * d ([hi 3C | lo 3C] in the pair layout), out per token [C];
//     n <= kTextMaxTokens, d <= kCausalMaxD
//   gelu16: exact-erf GELU, the shape of relu16
//   layernorm_f32: LayerNorm of 16-bit (or pair: hi + lo) rows into fp32 rows [tokens, C], C <= 1024
constexpr int kTextMaxTokens = 77;
constexpr int kCausalMaxD = 64;
cudaError_t text_embed(const int32_t* ids, int n, const float* tok, const float* pos, void* out, int C, bool bf16,
                       cudaStream_t s, bool split = false);
cudaError_t causal_attention(const void* qkv, int n, int heads, int d, void* out, bool bf16, cudaStream_t s, bool split = false);
cudaError_t gelu16(const void* in, void* out, long long n, bool bf16, cudaStream_t s, int split_c = 0);
cudaError_t layernorm_f32(const void* x, float* y, long long tokens, int C, const float* gamma, const float* beta, float eps,
                          bool bf16, cudaStream_t s, bool split = false);
// per-image (x - min) / (max - min) over HW fp32 values, in place; scratch: 2 uint32 per image.
// dmin: lower clamp of (max - min) (0 for the DPT readout, 1e-6 in ensemble_depth); zero_min: normalise by max only
cudaError_t minmax_normalize(float* x, int N, long long HW, unsigned int* scratch, cudaStream_t s, float dmin = 0.f, bool zero_min = false);
// out[HW] = median / mean over the B <= 32 members of d[B][HW] * scale[b] + shift[b]  (genpercept/util/ensemble.py)
cudaError_t ensemble_reduce(const float* d, int B, long long HW, const float* scale_dev, const float* shift_dev, bool median, float* out,
                            cudaStream_t s);

}  // namespace gp
