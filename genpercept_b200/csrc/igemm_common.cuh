// Device code shared by the two wgmma implicit-GEMM kernels (tap-streaming: igemm.cu, patch-resident:
// igemm_patch.cu): tile decoding, 16-bit helpers, the exact-erf GELU, the accumulator hand-off and the two epilogues.
//
// Both kernels run three warpgroups (384 threads, 1 CTA / SM): warps 0..3 epilogue, warps 4..7 the wgmma consumer
// (its fp32 accumulators live in registers during the K loop), warps 8..11 TMA producers.  At the end of a tile the
// consumer writes its accumulators into an fp32 tile in shared memory and starts the next tile's K loop while the
// epilogue warps read that tile one row per thread (tfull / tempty: single buffer, the registers are the second one).
// Patch-resident tiles at BN = 128 (p.acc_half) hand over in two 64-column halves through a 64-column shared tile: the
// consumer stores columns 0..63 and arrives tfull, waits tempty, stores columns 64..127 and arrives tfull again; the
// epilogue reads each half into registers and arrives tempty before it works on it.
//
// The consumer's K loop keeps one wgmma batch in flight: it commits batch k, waits until at most one batch is pending
// (batch k-1 retired) and only then releases the shared-memory stage that batch k-1 read.
//
// Registers: the producer warpgroup (warps 8..11, TMA issue only) drops to kProducerRegs per thread at its start and the
// epilogue and consumer warpgroups rise to kWorkerRegs (128 x 40 + 256 x 232 <= 64 K registers per SM), so the 128
// accumulators and the epilogue's 32-wide vectors fit without spilling.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "igemm.h"
#include "kernels.h"
#include "ptx.cuh"

namespace gp {
namespace {

constexpr int kABytes = kBM * kBK * 2;       // 16 KiB per 128-row tile
constexpr int kMaxSmem = 227 * 1024;
constexpr int kEpiWarps = 4;                 // warps 0..3
constexpr int kConsumerWarp0 = 4;            // warps 4..7: the wgmma warpgroup
constexpr int kRoleThreads = 384;
constexpr int kProducerRegs = 40;            // setmaxnreg: warps 8..11
constexpr int kWorkerRegs = 232;             // setmaxnreg: warps 0..7
static_assert(128 * kProducerRegs + 256 * kWorkerRegs <= 65536, "register file of one SM");

struct TileCoord {
  int n_tile, tx, ty, z0, z1;
};

__device__ __forceinline__ TileCoord decode_tile(const IgemmParams& p, int tile) {
  TileCoord t;
  t.n_tile = tile % p.n_tiles_n;
  int r = tile / p.n_tiles_n;
  t.tx = r % p.tiles_x;
  r /= p.tiles_x;
  t.ty = r % p.tiles_y;
  r /= p.tiles_y;
  t.z0 = r % p.Z0;
  t.z1 = r / p.Z0;
  return t;
}

// Tile row r -> pixel (x, y) inside the tile.  Tap-streaming tiles are TW x TH, row-major; patch-resident tiles are 8 x 8-pixel
// m64 blocks, TW / 8 of them across (igemm_patch.cu), so a warp's 32 rows there are an 8 x 4-pixel box.
__device__ __forceinline__ int2 tile_pixel(const IgemmParams& p, int r) {
  if (p.patch) {
    const int b = r >> 6, bx_bits = p.tw_shift - 3;
    return make_int2(((b & ((1 << bx_bits) - 1)) << 3) | (r & 7), ((b >> bx_bits) << 3) | ((r >> 3) & 7));
  }
  return make_int2(r & (p.TW - 1), r >> p.tw_shift);
}

template <bool BF16>
__device__ __forceinline__ float cvt16(uint16_t v) {
  if constexpr (BF16) {
    return __bfloat162float(__ushort_as_bfloat16(v));
  } else {
    return __half2float(__ushort_as_half(v));
  }
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
template <bool BF16>
__device__ __forceinline__ void add8(float* v, const uint4& u) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    v[2 * e] += cvt16<BF16>((uint16_t)(w[e] & 0xFFFF));
    v[2 * e + 1] += cvt16<BF16>((uint16_t)(w[e] >> 16));
  }
}

// 8 consecutive channels -> one 16-byte store; in the high-precision layout (lo != 0) the rounding residual
// v - float(hi) goes to the lo plane `lo` elements further.
template <bool BF16>
__device__ __forceinline__ void store8_hl(uint16_t* op, long long lo, const float* v) {
  uint4 u;
  u.x = pack16<BF16>(v[0], v[1]);
  u.y = pack16<BF16>(v[2], v[3]);
  u.z = pack16<BF16>(v[4], v[5]);
  u.w = pack16<BF16>(v[6], v[7]);
  *reinterpret_cast<uint4*>(op) = u;
  if (lo) {
    const uint32_t hw[4] = {u.x, u.y, u.z, u.w};
    uint32_t lw[4];
#pragma unroll
    for (int e = 0; e < 4; ++e)
      lw[e] = pack16<BF16>(v[2 * e] - cvt16<BF16>((uint16_t)(hw[e] & 0xFFFF)), v[2 * e + 1] - cvt16<BF16>((uint16_t)(hw[e] >> 16)));
    *reinterpret_cast<uint4*>(op + lo) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
  }
}

// ---------------------------------------------------------------- accumulator tile in shared memory
// fp32 [128 * MT rows][acc_pitch], acc_pitch = BN rounded up to 32; the 16-byte chunks of a row are XOR-swizzled by
// (row & 7) so that a warp reading eight consecutive rows one row per thread hits eight different bank groups.
__device__ __forceinline__ int acc_chunk(int ch, int row) { return (ch & ~7) | ((ch ^ row) & 7); }

// row `row`, columns c .. c + N - 1 (N = 16 or 32, c % 16 == 0) -> r[0 .. N-1]
template <int N>
__device__ __forceinline__ void acc_ld(const float* accs, int pitch, int row, int c, uint32_t (&r)[32]) {
  const float* rp = accs + (size_t)row * pitch;
#pragma unroll
  for (int q = 0; q < N / 4; ++q) {
    const float4 v = *reinterpret_cast<const float4*>(rp + (acc_chunk((c >> 2) + q, row) << 2));
    r[4 * q] = __float_as_uint(v.x); r[4 * q + 1] = __float_as_uint(v.y);
    r[4 * q + 2] = __float_as_uint(v.z); r[4 * q + 3] = __float_as_uint(v.w);
  }
}

template <int BN, bool BF16>
__device__ __forceinline__ void wgmma_ss(float (&d)[BN / 2], uint64_t a, uint64_t b, uint32_t acc) {
  if constexpr (BN == 16) wgmma_ss_n16<BF16>(d, a, b, acc);
  else if constexpr (BN == 32) wgmma_ss_n32<BF16>(d, a, b, acc);
  else if constexpr (BN == 64) wgmma_ss_n64<BF16>(d, a, b, acc);
  else wgmma_ss_n128<BF16>(d, a, b, acc);
}

// The consumer's register accumulators (MB m64 blocks: tile rows 64 mb ..) -> the shared tile.  wc: warp in the warpgroup.
// Columns 8 J0 .. 8 (J0 + NJ) - 1 of the accumulators land at tile columns 0 .. 8 NJ - 1 (a half-tile hand-off: J0 = 0 or 8,
// NJ = 8).
template <int BN, int MB, int J0 = 0, int NJ = BN / 8>
__device__ __forceinline__ void acc_store(float* accs, int pitch, float (&d)[MB][BN / 2], int wc, int lane) {
#pragma unroll
  for (int mb = 0; mb < MB; ++mb) {
    reg_fence(d[mb]);
#pragma unroll
    for (int j = J0; j < J0 + NJ; ++j)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int row = 64 * mb + 16 * wc + (lane >> 2) + 8 * hh, col = 8 * (j - J0) + 2 * (lane & 3);
        *reinterpret_cast<float2*>(accs + (size_t)row * pitch + (acc_chunk(col >> 2, row) << 2) + (col & 3)) =
            make_float2(d[mb][4 * j + 2 * hh], d[mb][4 * j + 2 * hh + 1]);
      }
  }
}

// gelu(g) = g * Phi(g), exact-erf form (what diffusers' GEGLU uses), with erf from Abramowitz-Stegun 7.1.26
// (|error| <= 1.5e-7): one MUFU.RCP, one MUFU.EX2 and a degree-5 Horner instead of erff()'s two-branch
// polynomial — the GEGLU projection is bound by its epilogue.
//   1 - erf(z) = (a1 t + ... + a5 t^5) e^{-z^2},  t = 1 / (1 + p z),  z = |g| / sqrt(2)
__device__ __forceinline__ float gelu_erf(float g) {
  const float z = fabsf(g) * 0.70710678118654752f;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.f)));
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(z * z * -1.4426950408889634f));
  float q = fmaf(1.061405429f, t, -1.453152027f);
  q = fmaf(q, t, 1.421413741f);
  q = fmaf(q, t, -0.284496736f);
  q = fmaf(q, t, 0.254829592f);
  q = q * t * e * 0.5f;                                   // = (1 - erf(z)) / 2 = Phi(-|g|)
  return g * (g >= 0.f ? 1.f - q : q);
}

__device__ __forceinline__ void epi_sync() {   // the epilogue threads only
  asm volatile("bar.sync 1, %0;" ::"n"(kEpiWarps * 32) : "memory");
}

// The bias of the CTA's current N tile lives in shared memory (kBiasSlots floats, zero beyond Cout): every 32-column piece
// of the epilogue would otherwise fetch it with eight dependent 16-byte global loads — with almost all of L1 configured as
// shared memory those miss to L2, in front of every piece.
constexpr int kBiasSlots = 288;
// A layer with several N tiles changes tile column on every tile of a CTA (tiles are numbered N-fastest and taken with a
// stride of gridDim.x), i.e. two barriers of all epilogue warps plus an L2 round trip per tile: when the padded Cout fits
// (p.bias_all, igemm_finalize) the whole bias vector is loaded once instead.
__device__ __forceinline__ void load_bias_tile(const IgemmParams& p, float* sbias, int n_base, int etid) {
  epi_sync();                                  // nobody still reads the previous tile's values
  const int count = p.bias_all ? p.bias_slots : kBiasSlots;
  for (int i = etid; i < count; i += kEpiWarps * 32) {
    const int n = n_base + i;
    sbias[i] = (p.bias != nullptr && n < p.Cout) ? __ldg(p.bias + n) : 0.f;
  }
  epi_sync();
}
__device__ __forceinline__ void bias32(const float* sbias, int c, float (&bz)[32]) {
#pragma unroll
  for (int q = 0; q < 32; q += 4) {
    const float4 b4 = *reinterpret_cast<const float4*>(sbias + c + q);
    bz[q] = b4.x; bz[q + 1] = b4.y; bz[q + 2] = b4.z; bz[q + 3] = b4.w;
  }
}

// Staged epilogue (shared by the tap-streaming and the patch-resident main loops): accumulator tile -> registers
// (bias / residuals / ReLU) -> 16-bit rows in a SWIZZLE_128B shared tile -> one TMA store per
// (warp, 64-channel group), plus the GroupNorm partial sums read back column-wise from the tile.
// SPLIT / RES are compile-time: with run-time flags every 32 x 64 piece pays the moves and branches around the variants
// not taken.  RES: 0 none, 1 residual tile through TMA, 2 per-thread rows.
template <bool BF16, bool SPLIT, int RES>
__device__ __forceinline__ void epilogue_staged(const IgemmParams& p, uint8_t* stg_base, float* sacc, float* sbias, uint64_t* tfull_bar,
                                                uint64_t* tempty_bar, uint64_t* res_bar, const float* accs, int warp, int lane) {
  // ===================================================================== epilogue, staged + TMA store
  // accumulator tile -> registers (bias / residuals / ReLU) -> 16-bit rows in a SWIZZLE_128B shared tile ->
  // one TMA store per (warp, 64-channel group): full-line writes instead of 16-byte pieces at a
  // 2C-byte stride, and image-edge clipping for free.  GroupNorm partial sums are read back
  // column-wise from the staged tile (conflict-free), in a fixed order.
  const int wq = warp;                       // tile rows [32*wq, +32)
  uint8_t* stg = stg_base + warp * 4096;
  const uint32_t stg_addr = smem_u32(stg);
  const uint32_t my_row = stg_addr + lane * 128;
  constexpr bool split = SPLIT;              // high-precision mode: a second staged tile (+kEpiWarps * 4 KiB) takes the lo plane
  const uint32_t my_row_lo = my_row + kEpiWarps * 4096;
  const int sw = lane & 7;
  uint32_t acc_phase = 0, res_phase = 0;
  const bool relu = (p.flags & IG_RELU) != 0;
  const bool do_stats = p.stats != nullptr;
  // half-tile hand-off (patch kernel, BN = 128, MT = 1): each 64-channel group is one hand-off of the consumer, the shared
  // tile holds that group only
  const bool halves = p.acc_half != 0;
  const int etid = threadIdx.x;
  int cur_img = -1;
  int cur_nt = -1;
  // Statistics scratch: sacc[warp][Cout] (mean, M2) and scnt[warp][64-channel group] the count behind them (the same for
  // every channel of a group: a warp sees the same rows for all of them).  Merge the four warps' records in a fixed
  // order, publish this CTA's slot, reset.
  auto scnt = [&](int i) -> float& { return sacc[kEpiWarps * 2 * p.Cout + i]; };   // derived, not kept live
  auto flush_stats = [&](int img) {
    epi_sync();
    float* dst = p.stats + ((long long)img * p.stats_slots + blockIdx.x) * p.Cout * kGnRec;
    for (int c = etid; c < p.Cout; c += kEpiWarps * 32) {
      float r[kEpiWarps][3];
#pragma unroll
      for (int w = 0; w < kEpiWarps; ++w) {
        r[w][0] = scnt(w * 8 + (c >> 6));
        r[w][1] = sacc[(w * p.Cout + c) * 2];
        r[w][2] = sacc[(w * p.Cout + c) * 2 + 1];
        sacc[(w * p.Cout + c) * 2] = 0.f; sacc[(w * p.Cout + c) * 2 + 1] = 0.f;
      }
      chan_merge(r[0][0], r[0][1], r[0][2], r[1][0], r[1][1], r[1][2]);
      chan_merge(r[2][0], r[2][1], r[2][2], r[3][0], r[3][1], r[3][2]);
      chan_merge(r[0][0], r[0][1], r[0][2], r[2][0], r[2][1], r[2][2]);
      dst[c * kGnRec] = r[0][0]; dst[c * kGnRec + 1] = r[0][1]; dst[c * kGnRec + 2] = r[0][2];
    }
    epi_sync();
    if (etid < kEpiWarps * 8) scnt(etid) = 0.f;
    epi_sync();
  };
  if (do_stats) {
    for (int i = etid; i < 8 * p.Cout + kEpiWarps * 8; i += kEpiWarps * 32) sacc[i] = 0.f;
    epi_sync();
  }
  if (p.bias_all) load_bias_tile(p, sbias, 0, etid);
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    const TileCoord t = decode_tile(p, tile);
    const int cls = p.cls_from_z0 ? t.z0 : 0;
    const int n_base = t.n_tile * p.BN;
    bool waited = false;   // whole-tile hand-off: tfull of this tile has been waited for
    if (t.n_tile != cur_nt && !p.bias_all) {
      load_bias_tile(p, sbias, n_base, etid);
      cur_nt = t.n_tile;
    }
    const int bias_origin = p.bias_all ? 0 : n_base;
    // The residual boxes of this CTA's NEXT tile are pulled into L2 now, a whole tile period before their TMA loads:
    // those loads sit serially in front of every 32 x 64 piece of the epilogue, and at DRAM latency under load four of
    // them per warp can outlast the main loop of the short-K (Cout = 128) layers.
    if (RES == 1 && lane == 0 && tile + (int)gridDim.x < p.total_tiles) {
      const TileCoord tn = decode_tile(p, tile + gridDim.x);
      const int ncls = p.cls_from_z0 ? tn.z0 : 0;
      for (int h = 0; h < p.MT; ++h) {
        const int2 o = tile_pixel(p, h * 128 + wq * 32);
        const int psx = tn.tx * p.TW + o.x, psy = tn.ty * p.TH + o.y;
        for (int c0 = 0; c0 < p.BN && tn.n_tile * p.BN + c0 < p.Cout; c0 += 64)
          tma_prefetch_l2_4d(&p.tmRes[ncls], tn.n_tile * p.BN + c0, psx, psy, tn.z1);
      }
    }
    if (do_stats) {
      const int img = p.stats_hw ? (t.tx * p.TW) / p.stats_hw : t.z1;
      if (img != cur_img) {
        if (cur_img >= 0) flush_stats(cur_img);
        cur_img = img;
      }
    }
    for (int h = 0; h < p.MT; ++h) {
      const int r0 = h * 128 + wq * 32;                       // first tile row of this warp
      const int row = r0 + lane;
      const int2 tp = tile_pixel(p, row), to = tile_pixel(p, r0);
      const int gy = t.ty * p.TH + tp.y, gx = t.tx * p.TW + tp.x;
      const bool valid = gy < p.gridH && gx < p.gridW;
      const int oy = gy * p.out_sy + p.cls_py[cls], ox = gx * p.out_sx + p.cls_px[cls];
      const long long pix_off = t.z1 * p.out_z1 + (long long)oy * p.out_row_stride + (long long)ox * p.out_pix_stride;
      const int sx = t.tx * p.TW + to.x, sy = t.ty * p.TH + to.y;   // store box origin
      for (int c0 = 0; c0 < p.BN; c0 += 64) {
        const int n0 = n_base + c0;
        if (n0 >= p.Cout) {
          if (!halves) break;
          mbar_wait(tfull_bar, acc_phase, 4);     // a half beyond Cout is handed over all the same
          mbar_arrive(tempty_bar);
          acc_phase ^= 1;
          continue;
        }
        if (lane == 0) tma_store_wait_read0();               // the previous store has finished reading the tile
        __syncwarp();
        uint4 rt[8];                                          // this thread's residual row (64 channels), res_tma only
        if constexpr (RES == 1) {
          if (lane == 0) {
            mbar_expect_tx(&res_bar[warp], 4096);
            tma_load_4d(stg, &p.tmRes[cls], &res_bar[warp], n0, sx, sy, t.z1);
          }
          mbar_wait(&res_bar[warp], res_phase, 7);
          res_phase ^= 1;
#pragma unroll
          for (int i = 0; i < 8; ++i)
            asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                         : "=r"(rt[i].x), "=r"(rt[i].y), "=r"(rt[i].z), "=r"(rt[i].w)
                         : "r"(my_row + ((i ^ sw) << 4)));
          __syncwarp();                                       // every row is in registers before the tile is overwritten
        }
        uint32_t rh[2][32];                                   // this row's accumulators of the two 32-column pieces
#pragma unroll
        for (int sub = 0; sub < 2; ++sub) {
          const int ns = n0 + sub * 32;
          const long long off = pix_off + ns;
          float bz[32];
          bias32(sbias, ns - bias_origin, bz);
          uint4 r1[4], r2[4];
          const bool has1 = RES == 1 || (RES == 2 && valid && p.res1 != nullptr), has2 = RES == 2 && valid && p.res2 != nullptr;
          if constexpr (RES == 1) {
#pragma unroll
            for (int q = 0; q < 4; ++q) r1[q] = rt[sub * 4 + q];
          } else if (has1) {
            const uint4* rp = reinterpret_cast<const uint4*>(reinterpret_cast<const uint16_t*>(p.res1) + off);
#pragma unroll
            for (int q = 0; q < 4; ++q) r1[q] = rp[q];
          }
          if (has2) {
            const uint4* rp = reinterpret_cast<const uint4*>(reinterpret_cast<const uint16_t*>(p.res2) + off);
#pragma unroll
            for (int q = 0; q < 4; ++q) r2[q] = rp[q];
          }
          if (halves) {
            if (sub == 0) {      // the whole half into registers: the consumer may store the next one while this one is worked on
              mbar_wait(tfull_bar, acc_phase, 4);
              acc_ld<32>(accs, p.acc_pitch, row, 0, rh[0]);
              acc_ld<32>(accs, p.acc_pitch, row, 32, rh[1]);
              mbar_arrive(tempty_bar);
              acc_phase ^= 1;
            }
          } else {
            if (!waited) {
              mbar_wait(tfull_bar, acc_phase, 4);
              waited = true;
            }
            acc_ld<32>(accs, p.acc_pitch, row, c0 + sub * 32, rh[sub]);
          }
          const uint32_t (&r)[32] = rh[sub];
          float v[32];
#pragma unroll
          for (int q = 0; q < 32; ++q) v[q] = __uint_as_float(r[q]) + bz[q];
          if (has1) {
#pragma unroll
            for (int q = 0; q < 4; ++q) add8<BF16>(&v[q * 8], r1[q]);
          }
          if (has2) {
#pragma unroll
            for (int q = 0; q < 4; ++q) add8<BF16>(&v[q * 8], r2[q]);
          }
          if (split) {       // lo planes of the residuals
            if (has1) {
              const uint4* rp = reinterpret_cast<const uint4*>(reinterpret_cast<const uint16_t*>(p.res1) + off + p.out_lo);
#pragma unroll
              for (int q = 0; q < 4; ++q) add8<BF16>(&v[q * 8], rp[q]);
            }
            if (has2) {
              const uint4* rp = reinterpret_cast<const uint4*>(reinterpret_cast<const uint16_t*>(p.res2) + off + p.out_lo);
#pragma unroll
              for (int q = 0; q < 4; ++q) add8<BF16>(&v[q * 8], rp[q]);
            }
          }
          if (relu) {
#pragma unroll
            for (int q = 0; q < 32; ++q) v[q] = fmaxf(v[q], 0.f);
          }
          if (!valid) {      // rows outside the image are clipped by the TMA store; zero them for the statistics
#pragma unroll
            for (int q = 0; q < 32; ++q) v[q] = 0.f;
          }
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const uint32_t a = my_row + (((sub * 4 + i) ^ sw) << 4);
            const uint32_t h0 = pack16<BF16>(v[8 * i], v[8 * i + 1]), h1 = pack16<BF16>(v[8 * i + 2], v[8 * i + 3]);
            const uint32_t h2 = pack16<BF16>(v[8 * i + 4], v[8 * i + 5]), h3 = pack16<BF16>(v[8 * i + 6], v[8 * i + 7]);
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(h0), "r"(h1), "r"(h2), "r"(h3) : "memory");
            if (split) {     // lo = v - float(hi), rounded to 16 bit
              const uint32_t hw[4] = {h0, h1, h2, h3};
              uint32_t lw[4];
#pragma unroll
              for (int e = 0; e < 4; ++e)
                lw[e] = pack16<BF16>(v[8 * i + 2 * e] - cvt16<BF16>((uint16_t)(hw[e] & 0xFFFF)),
                                     v[8 * i + 2 * e + 1] - cvt16<BF16>((uint16_t)(hw[e] >> 16)));
              const uint32_t al = my_row_lo + (((sub * 4 + i) ^ sw) << 4);
              asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(al), "r"(lw[0]), "r"(lw[1]), "r"(lw[2]), "r"(lw[3]) : "memory");
            }
          }
        }
        fence_proxy_async_shared();
        __syncwarp();
        if (lane == 0) {
          tma_store_4d(&p.tmOut[cls], stg_addr, n0, sx, sy, t.z1);
          if (split) tma_store_4d(&p.tmOutLo[cls], stg_addr + kEpiWarps * 4096, n0, sx, sy, t.z1);
          tma_store_commit();
        }
        if (do_stats) {
          // lane l owns channels n0 + 2l, n0 + 2l + 1: one 32-bit word per staged row.  The rows inside the image (bit rr
          // of `rows`) are summed as deviations from the first of them, which keeps the piece's M2 free of cancellation;
          // the piece's (count, mean, M2) is then merged into the warp's record.
          const uint32_t rows = __ballot_sync(0xffffffffu, valid);
          if (rows) {
            const uint32_t col = stg_addr + (lane & 3) * 4;
            const int chunk = lane >> 2;
            auto ld = [&](int rr, float& a, float& b) {
              uint32_t w;
              asm volatile("ld.shared.b32 %0, [%1];" : "=r"(w) : "r"(col + rr * 128 + ((chunk ^ (rr & 7)) << 4)));
              a = cvt16<BF16>((uint16_t)(w & 0xFFFF)); b = cvt16<BF16>((uint16_t)(w >> 16));
            };
            float k0, k1, s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;
            ld(__ffs(rows) - 1, k0, k1);
#pragma unroll 8
            for (int rr = 0; rr < 32; ++rr) {
              float a, b;
              ld(rr, a, b);
              const bool in = (rows >> rr) & 1u;
              a = in ? a - k0 : 0.f; b = in ? b - k1 : 0.f;
              s0 += a; q0 = fmaf(a, a, q0); s1 += b; q1 = fmaf(b, b, q1);
            }
            const float cnt = (float)__popc(rows), inv = __fdividef(1.f, cnt);
            float& cp = scnt(wq * 8 + (n0 >> 6));
            const float na = cp;
            float* d = sacc + ((size_t)wq * p.Cout + n0 + 2 * lane) * 2;
            float n_0 = na, n_1 = na;
            chan_merge(n_0, d[0], d[1], cnt, fmaf(s0, inv, k0), fmaxf(q0 - s0 * s0 * inv, 0.f));
            chan_merge(n_1, d[2], d[3], cnt, fmaf(s1, inv, k1), fmaxf(q1 - s1 * s1 * inv, 0.f));
            __syncwarp();
            if (lane == 0) cp = na + cnt;
            __syncwarp();
          }
        }
      }
    }
    if (!halves) {
      if (!waited) {
        mbar_wait(tfull_bar, acc_phase, 4);
      }
      mbar_arrive(tempty_bar);
      acc_phase ^= 1;
    }
  }
  if (lane == 0) tma_store_wait_read0();
  if (do_stats && cur_img >= 0) flush_stats(cur_img);
}


// Run-time flags -> the specialised staged epilogue.  LEAN (the patch-resident kernel): no (hi, lo) layout.
template <bool BF16, bool LEAN>
__device__ __forceinline__ void run_epilogue_staged(const IgemmParams& p, uint8_t* stg_base, float* sacc, float* sbias, uint64_t* tfull_bar,
                                                    uint64_t* tempty_bar, uint64_t* res_bar, const float* accs, int warp, int lane) {
  const int rm = p.res_tma ? 1 : ((p.res1 != nullptr || p.res2 != nullptr) ? 2 : 0);
  if constexpr (!LEAN) {
    if (p.out_lo != 0) {
      if (rm == 2) epilogue_staged<BF16, true, 2>(p, stg_base, sacc, sbias, tfull_bar, tempty_bar, res_bar, accs, warp, lane);
      else epilogue_staged<BF16, true, 0>(p, stg_base, sacc, sbias, tfull_bar, tempty_bar, res_bar, accs, warp, lane);
      return;
    }
  }
  if (rm == 1) epilogue_staged<BF16, false, 1>(p, stg_base, sacc, sbias, tfull_bar, tempty_bar, res_bar, accs, warp, lane);
  else if (rm == 2) epilogue_staged<BF16, false, 2>(p, stg_base, sacc, sbias, tfull_bar, tempty_bar, res_bar, accs, warp, lane);
  else epilogue_staged<BF16, false, 0>(p, stg_base, sacc, sbias, tfull_bar, tempty_bar, res_bar, accs, warp, lane);
}

// Direct epilogue: accumulator tile -> registers (bias / residuals / ReLU / affine clamp / GEGLU) -> global stores straight from
// the registers: fp32 NCHW maps, odd channel counts, GEGLU, the high-precision (hi, lo) layout.  No GroupNorm statistics:
// those are produced by the staged (TMA store) epilogue only.
// LEAN = the GEGLU projection of the default mode (full 32-column chunks, no residual, 16-bit output, no (hi, lo) planes): every
// other variant is compiled out of its loop (same reasoning as the staged epilogue's template parameters).
template <bool BF16, bool LEAN>
__device__ __forceinline__ void epilogue_direct(const IgemmParams& p, float* sbias, uint64_t* tfull_bar, uint64_t* tempty_bar,
                                                const float* accs, int warp, int lane) {
  // ===================================================================== epilogue
  const int wq = warp;                     // tile rows [32*wq, 32*wq+32)
  uint32_t acc_phase = 0;
  const bool f32out = !LEAN && (p.flags & IG_OUT_F32_NCHW) != 0;
  const bool relu = !LEAN && (p.flags & IG_RELU) != 0;
  const bool aff = !LEAN && (p.flags & IG_AFFINE_CLAMP01) != 0;
  const bool geglu = LEAN || (p.flags & IG_GEGLU) != 0;
  const void* const res1 = LEAN ? nullptr : p.res1;
  const void* const res2 = LEAN ? nullptr : p.res2;
  const long long out_lo = LEAN ? 0 : p.out_lo;
  const int etid = threadIdx.x;              // 0..127 among the epilogue threads
  int cur_nt = -1;
  if (p.bias_all) load_bias_tile(p, sbias, 0, etid);
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    const TileCoord t = decode_tile(p, tile);
    const int cls = p.cls_from_z0 ? t.z0 : 0;
    const int n_base = t.n_tile * p.BN;
    bool waited = false;
    if (t.n_tile != cur_nt && !p.bias_all) {
      load_bias_tile(p, sbias, n_base, etid);
      cur_nt = t.n_tile;
    }
    const int bias_origin = p.bias_all ? 0 : n_base;
    for (int h = 0; h < p.MT; ++h) {
      const int row = h * 128 + wq * 32 + lane;
      const int2 tp = tile_pixel(p, row);
      const int gy = t.ty * p.TH + tp.y, gx = t.tx * p.TW + tp.x;
      const bool valid = gy < p.gridH && gx < p.gridW;
      const int oy = gy * p.out_sy + p.cls_py[cls], ox = gx * p.out_sx + p.cls_px[cls];
      const long long pix_off = t.z1 * p.out_z1 + t.z0 * p.out_z0 + (long long)oy * p.out_row_stride +
                                (long long)ox * p.out_pix_stride;
      for (int c0 = 0; c0 < p.BN; c0 += 32) {
        const int ncols = (LEAN || p.BN - c0 >= 32) ? 32 : 16;
        const int n0 = n_base + c0;
        const int nvalid = LEAN ? 32 : min(ncols, p.Cout - n0);
        const bool live = valid && nvalid > 0;
        const long long off = pix_off + n0;
        // 16-byte accesses: the hi address and, in the (hi, lo) layout, the lo plane `out_lo` elements further
        const bool vec = !f32out && live && (nvalid == ncols) && ((off & 7) == 0) && ((out_lo & 7) == 0);
        // operands that do not depend on the accumulator are fetched BEFORE waiting on it
        float bz[32];
        bias32(sbias, n_base - bias_origin + c0, bz);
        uint4 r1[4], r2[4];
        const bool has1 = vec && res1 != nullptr, has2 = vec && res2 != nullptr;
        if (has1) {
          const uint4* rp = reinterpret_cast<const uint4*>(reinterpret_cast<const uint16_t*>(res1) + off);
#pragma unroll
          for (int q = 0; q < 4; ++q) if (q * 8 < ncols) r1[q] = rp[q];
        }
        if (has2) {
          const uint4* rp = reinterpret_cast<const uint4*>(reinterpret_cast<const uint16_t*>(res2) + off);
#pragma unroll
          for (int q = 0; q < 4; ++q) if (q * 8 < ncols) r2[q] = rp[q];
        }
        if (!waited) {
          mbar_wait(tfull_bar, acc_phase, 4);
          waited = true;
        }
        uint32_t r[32];
        if (LEAN || ncols == 32) acc_ld<32>(accs, p.acc_pitch, row, c0, r); else acc_ld<16>(accs, p.acc_pitch, row, c0, r);
        if (!live) continue;
        float v[32];
#pragma unroll
        for (int q = 0; q < 32; ++q) v[q] = __uint_as_float(r[q]) + bz[q];
        if (f32out) {
          float* o = reinterpret_cast<float*>(p.out);
#pragma unroll
          for (int q = 0; q < 32; ++q) {
            if (q < nvalid) {
              float x = v[q];
              if (relu) x = fmaxf(x, 0.f);
              if (aff) x = fminf(fmaxf((x + 1.f) * 0.5f, 0.f), 1.f);
              o[(((long long)t.z1 * p.Cout + (n0 + q)) * p.outH + oy) * p.outW + ox] = x;
            }
          }
          continue;
        }
        if (has1) {
#pragma unroll
          for (int q = 0; q < 4; ++q) if (q * 8 < ncols) add8<BF16>(&v[q * 8], r1[q]);
        } else if (res1 != nullptr && live) {
          const uint16_t* rp = reinterpret_cast<const uint16_t*>(res1) + off;
#pragma unroll
          for (int q = 0; q < 32; ++q) if (q < nvalid) v[q] += cvt16<BF16>(rp[q]);
        }
        if (has2) {
#pragma unroll
          for (int q = 0; q < 4; ++q) if (q * 8 < ncols) add8<BF16>(&v[q * 8], r2[q]);
        } else if (res2 != nullptr && live) {
          const uint16_t* rp = reinterpret_cast<const uint16_t*>(res2) + off;
#pragma unroll
          for (int q = 0; q < 32; ++q) if (q < nvalid) v[q] += cvt16<BF16>(rp[q]);
        }
        if (out_lo) {      // high-precision layout: lo planes of the residuals
#pragma unroll
          for (int ri = 0; ri < 2; ++ri) {
            const void* rb = ri == 0 ? res1 : res2;
            if (rb == nullptr || !live) continue;
            const uint16_t* rp = reinterpret_cast<const uint16_t*>(rb) + off + out_lo;
            if (vec) {
#pragma unroll
              for (int q = 0; q < 4; ++q) if (q * 8 < ncols) add8<BF16>(&v[q * 8], reinterpret_cast<const uint4*>(rp)[q]);
            } else {
#pragma unroll
              for (int q = 0; q < 32; ++q) if (q < nvalid) v[q] += cvt16<BF16>(rp[q]);
            }
          }
        }
        if (relu) {
#pragma unroll
          for (int q = 0; q < 32; ++q) v[q] = fmaxf(v[q], 0.f);
        }
        if (geglu) {   // [16 values | 16 gates] -> 16 outputs at column n0/2 (weights are packed interleaved)
          uint16_t* og = reinterpret_cast<uint16_t*>(p.out) + pix_off + (n0 >> 1);
          float g[16];
#pragma unroll
          for (int q = 0; q < 16; ++q) g[q] = v[q] * gelu_erf(v[16 + q]);
#pragma unroll
          for (int q = 0; q < 16; q += 8) store8_hl<BF16>(og + q, out_lo, &g[q]);
          continue;
        }
        uint16_t* op = reinterpret_cast<uint16_t*>(p.out) + off;
        if (vec) {
#pragma unroll
          for (int q = 0; q < 32; q += 8) {
            if (q < ncols) store8_hl<BF16>(op + q, out_lo, &v[q]);
          }
        } else if (live) {
#pragma unroll
          for (int q = 0; q < 32; ++q) {
            if (q < nvalid) {
              const uint16_t h = (uint16_t)(pack16<BF16>(v[q], 0.f) & 0xFFFF);
              op[q] = h;
              if (out_lo) op[q + out_lo] = (uint16_t)(pack16<BF16>(v[q] - cvt16<BF16>(h), 0.f) & 0xFFFF);
            }
          }
        }
      }
    }
    if (!waited) {   // unreachable (BN >= 16), kept so the barrier protocol can never desynchronise
      mbar_wait(tfull_bar, acc_phase, 4);
    }
    mbar_arrive(tempty_bar);
    acc_phase ^= 1;
  }
}

template <bool BF16>
__device__ __forceinline__ void run_epilogue_direct(const IgemmParams& p, float* sbias, uint64_t* tfull_bar, uint64_t* tempty_bar,
                                                    const float* accs, int warp, int lane) {
  const bool lean = (p.flags & IG_GEGLU) && !(p.flags & (IG_OUT_F32_NCHW | IG_RELU | IG_AFFINE_CLAMP01)) && p.out_lo == 0 &&
                    p.res1 == nullptr && p.res2 == nullptr && (p.BN % 32) == 0 && (p.Cout % p.BN) == 0;
  if (lean) epilogue_direct<BF16, true>(p, sbias, tfull_bar, tempty_bar, accs, warp, lane);
  else epilogue_direct<BF16, false>(p, sbias, tfull_bar, tempty_bar, accs, warp, lane);
}

}  // namespace
}  // namespace gp
