// Fused self-attention forward for head_dim 64 (the SD-2.1 UNet's BasicTransformerBlock.attn1):
//   O = softmax(Q K^T) V   per (image, head), non-causal, fp32 softmax state, 16-bit operands.
// (Softmax scale is folded into Wq at load.)  FlashAttention-style online softmax on wgmma; one 128-row query tile per
// CTA, shared by two consumer warpgroups of 64 rows each:
//
//   warp 8        : TMA producer — the Q tile once; K block [128 keys x 64] + V^T block [64 x 128 keys] per
//                   iteration into a 4-stage ring
//   warps 0..7    : two consumer warpgroups.  Per key block: S = Q K^T (wgmma m64n128k16 x 4, fp32 in registers),
//                   row max over the quad of threads that holds a row, P = 2^(s*c - m*c) rounded to 16 bit and fed
//                   straight from registers as the A operand of O += P V (wgmma m64n64k16 x 8); O is rescaled in
//                   registers whenever the running maximum grows.
//
// S and P never touch shared memory or HBM.
//
// SPLIT (the high-precision mode): every operand is an fp16 (hi, lo) pair.  The Q tile and each ring stage carry both
// planes (3 stages of K hi | K lo | V^T hi | V^T lo); S = Qh Kh^T + Ql Kh^T + Qh Kl^T in fp32, P is split in registers
// into ph = f16(p), pl = f16(p - ph), O += Ph Vh + Pl Vh + Ph Vl, and O is stored as its (hi, lo) pair.
#include "fattn.h"

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <utility>

#include "launch.h"
#include "ptx.cuh"

namespace gp {
namespace {

constexpr int kThreads = 288;                  // two consumer warpgroups + the producer warp
constexpr int kQBytes = 128 * 64 * 2;          // 16 KiB per plane
constexpr int kKBytes = 128 * 64 * 2;          // 16 KiB per plane
constexpr int kVBytes = 64 * 128 * 2;          // 16 KiB per plane (two 64-key sub-tiles of 8 KiB)
template <bool SPLIT> constexpr int kPlanesOf = SPLIT ? 2 : 1;
template <bool SPLIT> constexpr int kStagesOf = SPLIT ? 3 : 4;
template <bool SPLIT>
constexpr int kSmemBytes = kPlanesOf<SPLIT> * (kQBytes + kStagesOf<SPLIT> * (kKBytes + kVBytes)) + 256 + 1024;
static_assert(kSmemBytes<true> <= 227 * 1024, "shared memory of one CTA");

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
template <bool BF16>
__device__ __forceinline__ uint32_t pack16(float a, float b) {
  if constexpr (BF16) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  } else {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
}
// fp32 pair -> its fp16 (hi, lo) pairs: hi = f16(x), lo = f16(x - hi)
__device__ __forceinline__ void split16(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __half2 h = __floats2half2_rn(a, b);
  const float2 f = __half22float2(h);
  const __half2 l = __floats2half2_rn(a - f.x, b - f.y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

template <bool BF16, bool SPLIT>
__global__ void __launch_bounds__(kThreads, 1) fattn_kernel(const __grid_constant__ FattnParams p) {
  static_assert(!(BF16 && SPLIT), "the high-precision mode uses fp16 pairs");
  constexpr int PL = kPlanesOf<SPLIT>, kStages = kStagesOf<SPLIT>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;                               // [plane][16 KiB]
  uint8_t* sK = sQ + PL * kQBytes;                  // [stage][plane][16 KiB]
  uint8_t* sV = sK + kStages * PL * kKBytes;        // [stage][plane][16 KiB]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + kStages * PL * kVBytes);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;                     // [kStages]
  uint64_t* kv_empty = kv_full + kStages;           // [kStages]  one arrival per consumer warp

  const int warp = uniform_warp_id(), lane = threadIdx.x & 31;
  const int qt = blockIdx.x % p.q_tiles;
  const int bh = blockIdx.x / p.q_tiles;
  const int head = bh % p.heads, b = bh / p.heads;
  const int T = p.T;
  const int nblk = (T + 127) >> 7;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.tmQ);
    tma_prefetch_desc(&p.tmK);
    tma_prefetch_desc(&p.tmV);
    if constexpr (SPLIT) {
      tma_prefetch_desc(&p.tmQl);
      tma_prefetch_desc(&p.tmKl);
      tma_prefetch_desc(&p.tmVl);
    }
    mbar_init(q_full, 1);
    for (int i = 0; i < kStages; ++i) { mbar_init(&kv_full[i], 1); mbar_init(&kv_empty[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ------------------------------------------------------------------ TMA producer (whole warp waits, one lane issues)
    const bool leader = elect_one();
    if (leader) {
      mbar_expect_tx(q_full, (uint32_t)(PL * kQBytes));
      tma_load_3d(sQ, &p.tmQ, q_full, head * 64, qt * 128, b);
      if constexpr (SPLIT) tma_load_3d(sQ + kQBytes, &p.tmQl, q_full, head * 64, qt * 128, b);
    }
    for (int j = 0; j < nblk; ++j) {
      const int st = j % kStages;
      mbar_wait(&kv_empty[st], ((j / kStages) & 1) ^ 1, 10);
      if (leader) {
        mbar_expect_tx(&kv_full[st], PL * (kKBytes + kVBytes));
        uint8_t* k_st = sK + st * PL * kKBytes;
        uint8_t* v_st = sV + st * PL * kVBytes;
        tma_load_3d(k_st, &p.tmK, &kv_full[st], head * 64, j * 128, b);
        tma_load_3d(v_st, &p.tmV, &kv_full[st], j * 128, head * 64, b);
        tma_load_3d(v_st + 8192, &p.tmV, &kv_full[st], j * 128 + 64, head * 64, b);
        if constexpr (SPLIT) {
          tma_load_3d(k_st + kKBytes, &p.tmKl, &kv_full[st], head * 64, j * 128, b);
          tma_load_3d(v_st + kVBytes, &p.tmVl, &kv_full[st], j * 128, head * 64, b);
          tma_load_3d(v_st + kVBytes + 8192, &p.tmVl, &kv_full[st], j * 128 + 64, head * 64, b);
        }
      }
      __syncwarp();
    }
  } else if (warp < 8) {
    // ------------------------------------------------------------------ consumer warpgroup g: query rows 64 g .. 64 g + 63
    const int g = warp >> 2, wc = warp & 3;
    const float c2 = p.scale_log2e;
    const uint64_t q_desc = make_sw128_kmajor_desc(smem_u32(sQ + g * (kQBytes / 2)));
    float o[32];
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // rows r and r + 8 of this thread
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    mbar_wait(q_full, 0, 12);
    for (int j = 0; j < nblk; ++j) {
      const int st = j % kStages;
      mbar_wait(&kv_full[st], (j / kStages) & 1, 11);
      float s[64];
      const uint64_t k_desc = make_sw128_kmajor_desc(smem_u32(sK + st * PL * kKBytes));
      reg_fence(s);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_ss_n128<BF16>(s, q_desc + 2 * k, k_desc + 2 * k, k ? 1u : 0u);
      if constexpr (SPLIT) {   // + Ql Kh^T + Qh Kl^T  (descriptor addresses are in 16-byte units)
        constexpr uint64_t kQlo = kQBytes >> 4, kKlo = kKBytes >> 4;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          wgmma_ss_n128<false>(s, q_desc + kQlo + 2 * k, k_desc + 2 * k, 1u);
          wgmma_ss_n128<false>(s, q_desc + 2 * k, k_desc + kKlo + 2 * k, 1u);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(s);
      // s[4i + e]: key 8i + 2 (lane & 3) + (e & 1), row r (e < 2) or r + 8
      const int kvalid = T - j * 128;
      if (kvalid < 128) {
#pragma unroll
        for (int i = 0; i < 64; ++i)
          if (8 * (i >> 2) + 2 * (lane & 3) + (i & 1) >= kvalid) s[i] = -INFINITY;
      }
      float mx0 = m0, mx1 = m1;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        mx0 = fmaxf(mx0, fmaxf(s[4 * i], s[4 * i + 1]));
        mx1 = fmaxf(mx1, fmaxf(s[4 * i + 2], s[4 * i + 3]));
      }
      mx0 = quad_max(mx0);
      mx1 = quad_max(mx1);
      const float a0 = ex2((m0 - mx0) * c2), a1 = ex2((m1 - mx1) * c2);   // first block: m = -inf -> 0
      m0 = mx0;
      m1 = mx1;
      const float mb0 = m0 * c2, mb1 = m1 * c2;
      float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        s[4 * i] = ex2(fmaf(s[4 * i], c2, -mb0));
        s[4 * i + 1] = ex2(fmaf(s[4 * i + 1], c2, -mb0));
        s[4 * i + 2] = ex2(fmaf(s[4 * i + 2], c2, -mb1));
        s[4 * i + 3] = ex2(fmaf(s[4 * i + 3], c2, -mb1));
        ps0 += s[4 * i] + s[4 * i + 1];
        ps1 += s[4 * i + 2] + s[4 * i + 3];
      }
      l0 = l0 * a0 + ps0;
      l1 = l1 * a1 + ps1;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        o[4 * i] *= a0; o[4 * i + 1] *= a0;
        o[4 * i + 2] *= a1; o[4 * i + 3] *= a1;
      }
      // P as the register A operand: k step kk (keys 16 kk ..) = accumulator columns of n blocks 2 kk, 2 kk + 1
      const uint32_t v_base = smem_u32(sV + st * PL * kVBytes);
      reg_fence(o);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        const uint64_t v_desc = make_sw128_kmajor_desc(v_base + (kk >> 2) * 8192) + 2 * (kk & 3);
        if constexpr (SPLIT) {   // Ph Vh + Pl Vh + Ph Vl
          uint32_t ah[4], al[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) split16(s[8 * kk + 2 * e], s[8 * kk + 2 * e + 1], ah[e], al[e]);
          wgmma_rs_n64<false>(o, ah, v_desc, 1u);
          wgmma_rs_n64<false>(o, al, v_desc, 1u);
          wgmma_rs_n64<false>(o, ah, v_desc + (kVBytes >> 4), 1u);
        } else {
          const uint32_t a[4] = {pack16<BF16>(s[8 * kk], s[8 * kk + 1]), pack16<BF16>(s[8 * kk + 2], s[8 * kk + 3]),
                                 pack16<BF16>(s[8 * kk + 4], s[8 * kk + 5]), pack16<BF16>(s[8 * kk + 6], s[8 * kk + 7])};
          wgmma_rs_n64<BF16>(o, a, v_desc, 1u);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(o);
      __syncwarp();
      if (lane == 0) mbar_arrive(&kv_empty[st]);
    }
    // normalise, store: rows r and r + 8, columns 8 i + 2 (lane & 3) + {0, 1}
    const float inv0 = 1.f / quad_sum(l0), inv1 = 1.f / quad_sum(l1);
    const int r = qt * 128 + g * 64 + wc * 16 + (lane >> 2);
    uint16_t* ob = reinterpret_cast<uint16_t*>(p.out) + (long long)b * p.out_b_stride + head * 64 + 2 * (lane & 3);
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int row = r + 8 * hh;
      if (row >= T) continue;
      const float inv = hh ? inv1 : inv0;
      uint16_t* op = ob + (long long)row * p.out_row_stride;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if constexpr (SPLIT) {
          uint32_t hi, lo;
          split16(o[4 * i + 2 * hh] * inv, o[4 * i + 2 * hh + 1] * inv, hi, lo);
          *reinterpret_cast<uint32_t*>(op + 8 * i) = hi;
          *reinterpret_cast<uint32_t*>(op + p.out_lo + 8 * i) = lo;
        } else {
          *reinterpret_cast<uint32_t*>(op + 8 * i) = pack16<BF16>(o[4 * i + 2 * hh] * inv, o[4 * i + 2 * hh + 1] * inv);
        }
      }
    }
  }
}

}  // namespace

cudaError_t fattn_launch(const FattnParams& p, cudaStream_t stream) {
  static bool attr_dev[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
  if (!attr_dev[dev]) {      // function attributes are per device
    const std::pair<const void*, int> fns[3] = {{(const void*)fattn_kernel<false, false>, kSmemBytes<false>},
                                                {(const void*)fattn_kernel<true, false>, kSmemBytes<false>},
                                                {(const void*)fattn_kernel<false, true>, kSmemBytes<true>}};
    for (auto [f, bytes] : fns) {
      cudaError_t e = cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
      if (e != cudaSuccess) return e;
    }
    attr_dev[dev] = true;
  }
  const int grid = p.B * p.heads * p.q_tiles;
  if (grid <= 0) return cudaSuccess;
  if (p.split) launch(fattn_kernel<false, true>, grid, kThreads, kSmemBytes<true>, stream, p);
  else if (p.bf16) launch(fattn_kernel<true, false>, grid, kThreads, kSmemBytes<false>, stream, p);
  else launch(fattn_kernel<false, false>, grid, kThreads, kSmemBytes<false>, stream, p);
  return cudaGetLastError();
}

}  // namespace gp
