// Fused self-attention forward for one head of head_dim 512 (the VAE mid-block attention of the encoder and decoder):
//   O = softmax(Q K^T) V + b_v   per image, non-causal, fp32 softmax state, 16-bit operands.
// (Softmax scale is folded into Wq at load.)  The unfused path stores the whole T x T score matrix; here S and P never
// leave the SM, so the memory the op needs grows with T, not T^2.
//
// A 64 x 512 fp32 O tile is half the register file, so one CTA owns 64 query rows and splits O by columns:
//
//   warp 8        : TMA producer — the Q tile [64 x 512] once, then per 64-key block j the K block [64 keys x 512] and
//                   the V^T block [512 x 64 keys] as sixteen 8 KiB chunks (K d-chunks 0..7, V^T channel chunks 0..7)
//                   into a ring of sixteen slots, each with its own full / empty barrier.  K chunks of block j + 1 load
//                   while the consumers run softmax and P V of block j; V^T chunks of block j + 1 while they run
//                   Q K^T of block j + 1.
//   warps 0..7    : two consumer warpgroups over the same 64 rows.  Each computes the full S = Q K_j^T [64 x 64]
//                   (wgmma m64n64k16 x 32, fp32 in registers) and the identical online softmax, so P never has to be
//                   exchanged; warpgroup g then accumulates O[:, 256 g .. 256 g + 255] += P V_j (P from registers,
//                   wgmma m64n64k16 x 16) into 128 fp32 registers per thread.  Computing S twice costs half again
//                   the MMA work of the op; the loop is bound by the K / V^T traffic from L2, not by the tensor cores.
//
// fattn512_split_kernel is the high-precision mode's instance: every operand an fp16 (hi, lo) pair.  The Q tile holds
// both planes (128 KiB), which leaves room for six 16 KiB ring slots, each one d-chunk or channel chunk as its
// [hi | lo] pair.  Three producer warps feed three rings of two slots: warp 8 the K chunks both consumer warpgroups
// read, warps 9 and 10 the V^T chunks of consumer warpgroup 0 and 1.  Per key block, S = Qh Kh^T + Ql Kh^T + Qh Kl^T
// accumulates over the eight d-chunks (a chunk's slot is released as soon as its wgmma group retires); P is split in
// registers into ph = f16(p), pl = f16(p - ph) and O += Ph Vh + Pl Vh + Ph Vl, one channel chunk at a time.  The
// epilogue adds the to_v bias and stores O as its (hi, lo) pair.
#include "fattn512.h"

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <utility>

#include "launch.h"
#include "ptx.cuh"

namespace gp {
namespace {

constexpr int kThreads = 384;                  // two consumer warpgroups + the producer warpgroup (one warp issues)
constexpr int kChunk = 64 * 64 * 2;            // one 64 x 64 16-bit tile, 128-byte swizzled: 8 KiB
constexpr int kQBytes = 8 * kChunk;            // 64 query rows x 512
constexpr int kSlots = 16;
constexpr int kProducerRegs = 40;              // setmaxnreg: warps 8..11
constexpr int kConsumerRegs = 232;             // setmaxnreg: warps 0..7
static_assert(128 * kProducerRegs + 256 * kConsumerRegs <= 65536, "register file of one SM");                     // K block (8 chunks) + V^T block (8 chunks)
constexpr int kSmemBytes = kQBytes + kSlots * kChunk + 512 + 1024;

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

template <bool BF16>
__global__ void __launch_bounds__(kThreads, 1) fattn512_kernel(const __grid_constant__ Fattn512Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;                               // [8 chunks]
  uint8_t* sKV = sQ + kQBytes;                      // [kSlots chunks]: K d-chunks, then V^T channel chunks
  uint64_t* bars = reinterpret_cast<uint64_t*>(sKV + kSlots * kChunk);
  uint64_t* q_full = bars;
  uint64_t* full = bars + 1;                        // [kSlots]
  uint64_t* empty = full + kSlots;                  // [kSlots]  one arrival per consumer warp that reads the slot

  const int warp = uniform_warp_id(), lane = threadIdx.x & 31;
  const int qt = blockIdx.x % p.q_tiles;
  const int b = blockIdx.x / p.q_tiles;
  const int T = p.T;
  const int nblk = (T + 63) >> 6;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.tmQ);
    tma_prefetch_desc(&p.tmK);
    tma_prefetch_desc(&p.tmV);
    mbar_init(q_full, 1);
    for (int i = 0; i < kSlots; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], i < 8 ? 8 : 4);          // K chunks feed both warpgroups, a V^T chunk only one
    }
    fence_barrier_init();
  }
  __syncthreads();

  // The producer warpgroup hands registers to the consumers: 40 + 2 x 232 per thread fits the 64 Ki register file.  Each
  // warpgroup's role sits in its own branch after its setmaxnreg (ptxas ignores a setmaxnreg from which code of a larger
  // budget is reachable); warps 9..11 take part in the decrease and exit.
  if (warp < 8) {
    // ------------------------------------------------------------------ consumer warpgroup g: O columns 256 g .. 256 g + 255
    setmaxnreg_inc<kConsumerRegs>();
    const int g = warp >> 2, wc = warp & 3;
    const float c2 = p.scale_log2e;
    float o[4][32];                                 // o[n][4 i + e]: column 256 g + 64 n + 8 i + 2 (lane & 3) + (e & 1)
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // rows r and r + 8 of this thread
#pragma unroll
    for (int n = 0; n < 4; ++n)
#pragma unroll
      for (int i = 0; i < 32; ++i) o[n][i] = 0.f;
    mbar_wait(q_full, 0, 12);
    for (int j = 0; j < nblk; ++j) {
      const uint32_t par = j & 1;
      float s[32];
#pragma unroll 1
      for (int c = 0; c < 8; ++c) mbar_wait(&full[c], par, 11);
      reg_fence(s);
      wgmma_fence();
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const uint64_t q_desc = make_sw128_kmajor_desc(smem_u32(sQ + c * kChunk));
        const uint64_t k_desc = make_sw128_kmajor_desc(smem_u32(sKV + c * kChunk));
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_ss_n64<BF16>(s, q_desc + 2 * k, k_desc + 2 * k, (c | k) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(s);
      __syncwarp();
      if (lane == 0)
        for (int c = 0; c < 8; ++c) mbar_arrive(&empty[c]);
      // s[4i + e]: key 8i + 2 (lane & 3) + (e & 1), row r (e < 2) or r + 8
      const int kvalid = T - j * 64;
      if (kvalid < 64) {
#pragma unroll
        for (int i = 0; i < 32; ++i)
          if (8 * (i >> 2) + 2 * (lane & 3) + (i & 1) >= kvalid) s[i] = -INFINITY;
      }
      float mx0 = m0, mx1 = m1;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
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
      for (int i = 0; i < 8; ++i) {
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
      for (int n = 0; n < 4; ++n)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          o[n][4 * i] *= a0; o[n][4 * i + 1] *= a0;
          o[n][4 * i + 2] *= a1; o[n][4 * i + 3] *= a1;
        }
      // P as the register A operand: k step kk (keys 16 kk ..) = accumulator columns of n blocks 2 kk, 2 kk + 1.
      // B = this warpgroup's four V^T channel chunks (slots 8 + 4 g + n), keys 16 kk .. at +32 bytes per k step.
      uint32_t a[4][4];
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
#pragma unroll
        for (int e = 0; e < 4; ++e) a[kk][e] = pack16<BF16>(s[8 * kk + 2 * e], s[8 * kk + 2 * e + 1]);
#pragma unroll 1
      for (int n = 0; n < 4; ++n) mbar_wait(&full[8 + 4 * g + n], par, 13);
      const uint32_t v_base = smem_u32(sKV + (8 + 4 * g) * kChunk);
#pragma unroll
      for (int n = 0; n < 4; ++n) reg_fence(o[n]);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
#pragma unroll
        for (int n = 0; n < 4; ++n)
          wgmma_rs_n64<BF16>(o[n], a[kk], make_sw128_kmajor_desc(v_base + n * kChunk) + 2 * kk, 1u);
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int n = 0; n < 4; ++n) reg_fence(o[n]);
      __syncwarp();
      if (lane == 0)
        for (int n = 0; n < 4; ++n) mbar_arrive(&empty[8 + 4 * g + n]);
    }
    // normalise, add the bias, store: rows r and r + 8, columns 256 g + 64 n + 8 i + 2 (lane & 3) + {0, 1}
    const float inv0 = 1.f / quad_sum(l0), inv1 = 1.f / quad_sum(l1);
    const int r = qt * 64 + wc * 16 + (lane >> 2);
    const int col0 = 256 * g + 2 * (lane & 3);
    uint16_t* ob = reinterpret_cast<uint16_t*>(p.out) + (long long)b * p.out_b_stride + col0;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int row = r + 8 * hh;
      if (row >= T) continue;
      const float inv = hh ? inv1 : inv0;
      uint16_t* op = ob + (long long)row * p.out_row_stride;
#pragma unroll
      for (int n = 0; n < 4; ++n)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          float2 bv = make_float2(0.f, 0.f);
          if (p.bias) bv = *reinterpret_cast<const float2*>(p.bias + col0 + 64 * n + 8 * i);
          *reinterpret_cast<uint32_t*>(op + 64 * n + 8 * i) =
              pack16<BF16>(o[n][4 * i + 2 * hh] * inv + bv.x, o[n][4 * i + 2 * hh + 1] * inv + bv.y);
        }
    }
    return;
  }
  setmaxnreg_dec<kProducerRegs>();
  if (warp == 8) {
    // ------------------------------------------------------------------ TMA producer (whole warp waits, one lane issues)
    const bool leader = elect_one();
    if (leader) {
      mbar_expect_tx(q_full, (uint32_t)kQBytes);
      for (int c = 0; c < 8; ++c) tma_load_3d(sQ + c * kChunk, &p.tmQ, q_full, c * 64, qt * 64, b);
    }
    for (int j = 0; j < nblk; ++j) {
      for (int s = 0; s < kSlots; ++s) {
        mbar_wait(&empty[s], (j & 1) ^ 1, 10);
        if (leader) {
          mbar_expect_tx(&full[s], (uint32_t)kChunk);
          if (s < 8) tma_load_3d(sKV + s * kChunk, &p.tmK, &full[s], s * 64, j * 64, b);
          else tma_load_3d(sKV + s * kChunk, &p.tmV, &full[s], j * 64, (s - 8) * 64, b);
        }
        __syncwarp();
      }
    }
  }
}

constexpr int kPair = 2 * kChunk;              // one chunk's [hi | lo] planes: 16 KiB
constexpr int kRingSlots = 2;                  // per ring: K, V^T of warpgroup 0, V^T of warpgroup 1
constexpr int kSplitSmemBytes = 2 * kQBytes + 3 * kRingSlots * kPair + 256 + 1024;
static_assert(kSplitSmemBytes <= 227 * 1024, "shared memory of one CTA");

__global__ void __launch_bounds__(kThreads, 1) fattn512_split_kernel(const __grid_constant__ Fattn512Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;                               // [8 hi chunks | 8 lo chunks]
  uint8_t* sK = sQ + 2 * kQBytes;                   // [kRingSlots pairs]
  uint8_t* sV = sK + kRingSlots * kPair;            // [warpgroup][kRingSlots pairs]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + 2 * kRingSlots * kPair);
  uint64_t* q_full = bars;
  uint64_t* k_full = bars + 1;                      // [kRingSlots]
  uint64_t* k_empty = k_full + kRingSlots;          // [kRingSlots]  one arrival per consumer warp (8)
  uint64_t* v_full = k_empty + kRingSlots;          // [warpgroup][kRingSlots]
  uint64_t* v_empty = v_full + 2 * kRingSlots;      // [warpgroup][kRingSlots]  one arrival per warp of that warpgroup (4)

  const int warp = uniform_warp_id(), lane = threadIdx.x & 31;
  const int qt = blockIdx.x % p.q_tiles;
  const int b = blockIdx.x / p.q_tiles;
  const int T = p.T;
  const int nblk = (T + 63) >> 6;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.tmQ);
    tma_prefetch_desc(&p.tmK);
    tma_prefetch_desc(&p.tmV);
    tma_prefetch_desc(&p.tmQl);
    tma_prefetch_desc(&p.tmKl);
    tma_prefetch_desc(&p.tmVl);
    mbar_init(q_full, 1);
    for (int i = 0; i < kRingSlots; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&k_empty[i], 8);
    }
    for (int i = 0; i < 2 * kRingSlots; ++i) {
      mbar_init(&v_full[i], 1);
      mbar_init(&v_empty[i], 4);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 8) {
    // ------------------------------------------------------------------ consumer warpgroup g: O columns 256 g .. 256 g + 255
    setmaxnreg_inc<kConsumerRegs>();
    const int g = warp >> 2, wc = warp & 3;
    const float c2 = p.scale_log2e;
    uint64_t* vf = v_full + g * kRingSlots;
    uint64_t* ve = v_empty + g * kRingSlots;
    const uint32_t v_base = smem_u32(sV + g * kRingSlots * kPair);
    float o[4][32];                                 // o[n][4 i + e]: column 256 g + 64 n + 8 i + 2 (lane & 3) + (e & 1)
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // rows r and r + 8 of this thread
#pragma unroll
    for (int n = 0; n < 4; ++n)
#pragma unroll
      for (int i = 0; i < 32; ++i) o[n][i] = 0.f;
    mbar_wait(q_full, 0, 12);
    for (int j = 0; j < nblk; ++j) {
      float s[32];
      reg_fence(s);
      // S over the eight d-chunks; K chunk c of block j is ring entry 8 j + c
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const int slot = c % kRingSlots;
        mbar_wait(&k_full[slot], ((8 * j + c) / kRingSlots) & 1, 11);
        const uint64_t qh = make_sw128_kmajor_desc(smem_u32(sQ + c * kChunk));
        const uint64_t ql = make_sw128_kmajor_desc(smem_u32(sQ + kQBytes + c * kChunk));
        const uint64_t kh = make_sw128_kmajor_desc(smem_u32(sK + slot * kPair));
        const uint64_t kl = kh + (kChunk >> 4);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          wgmma_ss_n64<false>(s, qh + 2 * k, kh + 2 * k, (c | k) ? 1u : 0u);
          wgmma_ss_n64<false>(s, ql + 2 * k, kh + 2 * k, 1u);
          wgmma_ss_n64<false>(s, qh + 2 * k, kl + 2 * k, 1u);
        }
        wgmma_commit();
        if (c > 0) {
          wgmma_wait<1>();
          __syncwarp();
          if (lane == 0) mbar_arrive(&k_empty[(c - 1) % kRingSlots]);
        }
      }
      wgmma_wait<0>();
      reg_fence(s);
      __syncwarp();
      if (lane == 0) mbar_arrive(&k_empty[7 % kRingSlots]);
      // s[4i + e]: key 8i + 2 (lane & 3) + (e & 1), row r (e < 2) or r + 8
      const int kvalid = T - j * 64;
      if (kvalid < 64) {
#pragma unroll
        for (int i = 0; i < 32; ++i)
          if (8 * (i >> 2) + 2 * (lane & 3) + (i & 1) >= kvalid) s[i] = -INFINITY;
      }
      float mx0 = m0, mx1 = m1;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
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
      for (int i = 0; i < 8; ++i) {
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
      for (int n = 0; n < 4; ++n)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          o[n][4 * i] *= a0; o[n][4 * i + 1] *= a0;
          o[n][4 * i + 2] *= a1; o[n][4 * i + 3] *= a1;
        }
      // P as the register A operand, k step kk (keys 16 kk ..) = accumulator columns of n blocks 2 kk, 2 kk + 1
      uint32_t ah[4][4], al[4][4];
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
#pragma unroll
        for (int e = 0; e < 4; ++e) split16(s[8 * kk + 2 * e], s[8 * kk + 2 * e + 1], ah[kk][e], al[kk][e]);
#pragma unroll
      for (int n = 0; n < 4; ++n) reg_fence(o[n]);
      // O[:, 64 n ..] += P V^T chunk n of this warpgroup; chunk n of block j is ring entry 4 j + n
#pragma unroll
      for (int n = 0; n < 4; ++n) {
        const int slot = n % kRingSlots;
        mbar_wait(&vf[slot], ((4 * j + n) / kRingSlots) & 1, 13);
        const uint64_t vh = make_sw128_kmajor_desc(v_base + slot * kPair);
        const uint64_t vl = vh + (kChunk >> 4);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          wgmma_rs_n64<false>(o[n], ah[kk], vh + 2 * kk, 1u);
          wgmma_rs_n64<false>(o[n], al[kk], vh + 2 * kk, 1u);
          wgmma_rs_n64<false>(o[n], ah[kk], vl + 2 * kk, 1u);
        }
        wgmma_commit();
        if (n > 0) {
          wgmma_wait<1>();
          __syncwarp();
          if (lane == 0) mbar_arrive(&ve[(n - 1) % kRingSlots]);
        }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int n = 0; n < 4; ++n) reg_fence(o[n]);
      __syncwarp();
      if (lane == 0) mbar_arrive(&ve[3 % kRingSlots]);
    }
    // normalise, add the bias, store hi and lo: rows r and r + 8, columns 256 g + 64 n + 8 i + 2 (lane & 3) + {0, 1}
    const float inv0 = 1.f / quad_sum(l0), inv1 = 1.f / quad_sum(l1);
    const int r = qt * 64 + wc * 16 + (lane >> 2);
    const int col0 = 256 * g + 2 * (lane & 3);
    uint16_t* ob = reinterpret_cast<uint16_t*>(p.out) + (long long)b * p.out_b_stride + col0;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int row = r + 8 * hh;
      if (row >= T) continue;
      const float inv = hh ? inv1 : inv0;
      uint16_t* op = ob + (long long)row * p.out_row_stride;
#pragma unroll
      for (int n = 0; n < 4; ++n)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          float2 bv = make_float2(0.f, 0.f);
          if (p.bias) bv = *reinterpret_cast<const float2*>(p.bias + col0 + 64 * n + 8 * i);
          uint32_t hi, lo;
          split16(o[n][4 * i + 2 * hh] * inv + bv.x, o[n][4 * i + 2 * hh + 1] * inv + bv.y, hi, lo);
          *reinterpret_cast<uint32_t*>(op + 64 * n + 8 * i) = hi;
          *reinterpret_cast<uint32_t*>(op + p.out_lo + 64 * n + 8 * i) = lo;
        }
    }
    return;
  }
  setmaxnreg_dec<kProducerRegs>();
  // ------------------------------------------------------------------ TMA producers (whole warp waits, one lane issues)
  const bool leader = elect_one();
  if (warp == 8) {   // Q once, then the K ring
    if (leader) {
      mbar_expect_tx(q_full, (uint32_t)(2 * kQBytes));
      for (int c = 0; c < 8; ++c) {
        tma_load_3d(sQ + c * kChunk, &p.tmQ, q_full, c * 64, qt * 64, b);
        tma_load_3d(sQ + kQBytes + c * kChunk, &p.tmQl, q_full, c * 64, qt * 64, b);
      }
    }
    for (int j = 0; j < nblk; ++j)
      for (int c = 0; c < 8; ++c) {
        const int n = 8 * j + c, slot = n % kRingSlots;
        mbar_wait(&k_empty[slot], ((n / kRingSlots) & 1) ^ 1, 10);
        if (leader) {
          uint8_t* dst = sK + slot * kPair;
          mbar_expect_tx(&k_full[slot], (uint32_t)kPair);
          tma_load_3d(dst, &p.tmK, &k_full[slot], c * 64, j * 64, b);
          tma_load_3d(dst + kChunk, &p.tmKl, &k_full[slot], c * 64, j * 64, b);
        }
        __syncwarp();
      }
  } else if (warp == 9 || warp == 10) {   // the V^T ring of consumer warpgroup g: its channel chunks 4 g .. 4 g + 3
    const int g = warp - 9;
    uint64_t* vf = v_full + g * kRingSlots;
    uint64_t* ve = v_empty + g * kRingSlots;
    for (int j = 0; j < nblk; ++j)
      for (int c = 0; c < 4; ++c) {
        const int n = 4 * j + c, slot = n % kRingSlots;
        mbar_wait(&ve[slot], ((n / kRingSlots) & 1) ^ 1, 10);
        if (leader) {
          uint8_t* dst = sV + (g * kRingSlots + slot) * kPair;
          mbar_expect_tx(&vf[slot], (uint32_t)kPair);
          tma_load_3d(dst, &p.tmV, &vf[slot], j * 64, (4 * g + c) * 64, b);
          tma_load_3d(dst + kChunk, &p.tmVl, &vf[slot], j * 64, (4 * g + c) * 64, b);
        }
        __syncwarp();
      }
  }
}

}  // namespace

cudaError_t fattn512_launch(const Fattn512Params& p, cudaStream_t stream) {
  static bool attr_dev[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
  if (!attr_dev[dev]) {      // function attributes are per device
    const std::pair<const void*, int> fns[3] = {{(const void*)fattn512_kernel<false>, kSmemBytes},
                                                {(const void*)fattn512_kernel<true>, kSmemBytes},
                                                {(const void*)fattn512_split_kernel, kSplitSmemBytes}};
    for (auto [f, bytes] : fns) {
      cudaError_t e = cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
      if (e != cudaSuccess) return e;
    }
    attr_dev[dev] = true;
  }
  const long long grid = (long long)p.B * p.q_tiles;
  if (grid <= 0) return cudaSuccess;
  if (grid > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
  if (p.split) launch(fattn512_split_kernel, (int)grid, kThreads, kSplitSmemBytes, stream, p);
  else if (p.bf16) launch(fattn512_kernel<true>, (int)grid, kThreads, kSmemBytes, stream, p);
  else launch(fattn512_kernel<false>, (int)grid, kThreads, kSmemBytes, stream, p);
  return cudaGetLastError();
}

}  // namespace gp
