// wgmma implicit-GEMM kernel (see igemm.h for the operand model).
//
// Warp roles (384 threads, 1 CTA / SM, persistent over a static round-robin tile list; see igemm_common.cuh):
//   warps 0..3  : epilogue (accumulator tile -> bias / residual / act -> staged tile -> TMA store, GroupNorm partial sums)
//   warps 4..7  : wgmma consumer: per 64-channel K block, 4 x (MT * 2) wgmma m64 x BN x 16 from the stage's A and B boxes
//   warp 8      : TMA producer A (activation box per 64-channel K block, `stages`-deep ring)
//   warp 11     : TMA producer B (weight box per K block)
// MT = 2 (a 256-pixel M tile per CTA sharing every weight box) when BN <= 64: the consumer holds MT * 128 x BN fp32
// accumulators in registers, at most 128 per thread.
#include "igemm.h"

#include <cstring>

#include "igemm_common.cuh"
#include "launch.h"

namespace gp {

namespace {

// K loop of the tap-streaming kernel for one (BN, MB = 2 * MT) instance; the whole consumer warpgroup runs it.
// One batch (the wgmmas of one K block) stays in flight: batch kb is committed before batch kb - 1 is waited for, and
// batch kb - 1's stage is released only then.  The ring holds >= 2 stages (igemm_finalize), so the stage kb waits for is
// never the one still held.  Batches into one accumulator run in issue order: the summation order is unchanged.
template <bool BF16, int BN, int MB>
__device__ __forceinline__ void tap_consumer(const IgemmParams& p, uint8_t* smem, int stage_bytes, int a_bytes, float* accs,
                                             uint64_t* full_bar, uint64_t* empty_bar, uint64_t* tfull_bar, uint64_t* tempty_bar,
                                             int wc, int lane) {
  float d[MB][BN / 2];
  int stage = 0;
  uint32_t phase = 0, acc_phase = 0;
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    const TileCoord t = decode_tile(p, tile);
    const int cls = p.cls_from_z0 ? t.z0 : 0;
    const int nkb = p.nkb[cls] * p.npass;
    int held = -1;                                  // stage read by the batch still in flight
    for (int kb = 0; kb < nkb; ++kb) {
      mbar_wait(&full_bar[stage], phase, 3);
      const uint32_t a_addr = smem_u32(smem + stage * stage_bytes);
      const uint64_t b_desc = make_sw128_kmajor_desc(a_addr + a_bytes);
#pragma unroll
      for (int mb = 0; mb < MB; ++mb) reg_fence(d[mb]);
      wgmma_fence();
#pragma unroll
      for (int mb = 0; mb < MB; ++mb) {
        const uint64_t a_desc = make_sw128_kmajor_desc(a_addr + mb * (kABytes / 2));
#pragma unroll
        for (int k = 0; k < kBK / 16; ++k)   // +32 bytes per K step inside the 128-byte swizzle row -> +2 in the (addr >> 4) field
          wgmma_ss<BN, BF16>(d[mb], a_desc + 2 * k, b_desc + 2 * k, (kb | k) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<1>();                              // batch kb - 1 has retired
#pragma unroll
      for (int mb = 0; mb < MB; ++mb) reg_fence(d[mb]);
      if (held >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[held]);
      }
      held = stage;
      if (++stage == p.stages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int mb = 0; mb < MB; ++mb) reg_fence(d[mb]);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[held]);
    mbar_wait(tempty_bar, acc_phase ^ 1, 2);     // the epilogue has read the previous tile
    acc_store<BN, MB>(accs, p.acc_pitch, d, wc, lane);
    mbar_arrive(tfull_bar);
    acc_phase ^= 1;
  }
}

template <bool BF16>
__device__ __forceinline__ void run_tap_consumer(const IgemmParams& p, uint8_t* smem, int stage_bytes, int a_bytes, float* accs,
                                                 uint64_t* full_bar, uint64_t* empty_bar, uint64_t* tfull_bar, uint64_t* tempty_bar,
                                                 int wc, int lane) {
#define GP_TAP(BN_, MB_) tap_consumer<BF16, BN_, MB_>(p, smem, stage_bytes, a_bytes, accs, full_bar, empty_bar, tfull_bar, tempty_bar, wc, lane)
  if (p.MT == 2) {
    if (p.BN == 16) GP_TAP(16, 4); else if (p.BN == 32) GP_TAP(32, 4); else GP_TAP(64, 4);
  } else {
    if (p.BN == 16) GP_TAP(16, 2); else if (p.BN == 32) GP_TAP(32, 2); else if (p.BN == 64) GP_TAP(64, 2); else GP_TAP(128, 2);
  }
#undef GP_TAP
}

template <bool BF16>
__global__ void __launch_bounds__(kRoleThreads, 1) igemm_kernel(const __grid_constant__ IgemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int a_bytes = kABytes * p.MT;
  const int stage_bytes = a_bytes + p.BN * 128;
  const int stages = p.stages;
  uint8_t* stg_base = smem + stages * stage_bytes;                     // one 4 KiB staging tile per epilogue warp (tma_store only)
  float* accs = reinterpret_cast<float*>(stg_base + (p.tma_store ? (p.out_lo ? 2 : 1) * kEpiWarps * 4096 : 0));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(accs + 128 * p.MT * p.acc_pitch);
  uint64_t* empty_bar = full_bar + stages;
  uint64_t* tfull_bar = empty_bar + stages;
  uint64_t* tempty_bar = tfull_bar + 1;
  uint64_t* res_bar = tempty_bar + 1;                                  // [epilogue warps] residual tile landed
  float* sbias = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(res_bar + kEpiWarps) + 15) & ~uintptr_t(15));   // [bias_slots]
  float* sacc = sbias + p.bias_slots;   // [4 epilogue warps][Cout][2] + [4][8] counts, only with p.stats

  const int warp = uniform_warp_id();
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int i = 0; i < (p.npass > 1 ? 8 : 4); ++i) tma_prefetch_desc(&p.tmA[i]);
    tma_prefetch_desc(&p.tmB);
    for (int i = 0; i < stages; ++i) {
      mbar_init(&full_bar[i], 2);    // producer A + producer B
      mbar_init(&empty_bar[i], 4);   // the four consumer warps
    }
    mbar_init(tfull_bar, 128);
    mbar_init(tempty_bar, kEpiWarps * 32);
    for (int i = 0; i < kEpiWarps; ++i) mbar_init(&res_bar[i], 1);
    fence_barrier_init();
  }
  __syncthreads();

  // The producer warpgroup gives registers to the other two (igemm_common.cuh).  Each warpgroup's roles sit in their own
  // branch after its setmaxnreg (ptxas ignores a setmaxnreg from which code of a larger budget is reachable); warps 9 and
  // 10 take part in the decrease and exit.
  if (warp < 8) {
    setmaxnreg_inc<kWorkerRegs>();
    if (warp >= kConsumerWarp0) {
      // ===================================================================== wgmma consumer
      run_tap_consumer<BF16>(p, smem, stage_bytes, a_bytes, accs, full_bar, empty_bar, tfull_bar, tempty_bar, warp - kConsumerWarp0, lane);
    } else {
      // ===================================================================== epilogue
      if (p.tma_store) run_epilogue_staged<BF16, false>(p, stg_base, sacc, sbias, tfull_bar, tempty_bar, res_bar, accs, warp, lane);
      else run_epilogue_direct<BF16>(p, sbias, tfull_bar, tempty_bar, accs, warp, lane);
    }
    return;
  }
  setmaxnreg_dec<kProducerRegs>();

  // Single-thread roles run warp-uniform (every lane walks the loop and waits on the barriers) and one
  // elected lane issues: the TMA coordinates then stay in uniform registers.
  if (warp == 8) {
    // ===================================================================== TMA producer A
    const bool leader = elect_one();
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const TileCoord t = decode_tile(p, tile);
      const int cls = p.cls_from_z0 ? t.z0 : 0;
      const int a_n = t.z1 * p.a_n_z1 + t.z0 * p.a_n_z0;
      const int a_k0 = t.z0 * p.a_k_z0;
      const int x0 = t.tx * p.TW, y0 = t.ty * p.TH;
      const int ns = p.nseg[cls];
      for (int pass = 0; pass < p.npass; ++pass) {
        const int moff = p.pass_amap[pass];
        for (int s = 0; s < ns; ++s) {
          const IgemmSeg sg = p.seg[cls][s];
          const CUtensorMap* tm = &p.tmA[sg.map + moff];
          const int xs = x0 + sg.dx, ys = y0 + sg.dy;
          for (int c = 0; c < sg.nchunks; ++c) {
            mbar_wait(&empty_bar[stage], phase ^ 1, 1);
            if (leader) {
              mbar_expect_tx(&full_bar[stage], (uint32_t)a_bytes);
              tma_load_4d(smem + stage * stage_bytes, tm, &full_bar[stage], a_k0 + c * kBK, xs, ys, a_n);
            }
            __syncwarp();
            if (++stage == stages) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else if (warp == 11) {
    // ===================================================================== TMA producer B
    const bool leader = elect_one();
    int stage = 0;
    uint32_t phase = 0;
    const uint32_t b_bytes = (uint32_t)p.BN * 128;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const TileCoord t = decode_tile(p, tile);
      const int cls = p.cls_from_z0 ? t.z0 : 0;
      const int b_z = t.z1 * p.b_z_z1 + t.z0 * p.b_z_z0;
      const int b_row = t.z0 * p.b_row_z0 + t.n_tile * p.BN;
      const int b_k0 = t.z0 * p.b_k_z0;
      const int nkb = p.nkb[cls];
      for (int pass = 0; pass < p.npass; ++pass) {
        const CUtensorMap* tmb = p.pass_bmap[pass] ? &p.tmB2 : &p.tmB;
        const int bk = b_k0 + p.pass_bk[pass];
        for (int kb = 0; kb < nkb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1, 5);
          if (leader) {
            mbar_expect_tx(&full_bar[stage], b_bytes);
            tma_load_3d(smem + stage * stage_bytes + a_bytes, tmb, &full_bar[stage], bk + kb * kBK, b_row, b_z);
          }
          __syncwarp();
          if (++stage == stages) { stage = 0; phase ^= 1; }
        }
      }
    }
  }
}

}  // namespace

namespace {

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                    CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                    CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (fn) return fn;
  void* f = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess ||
      q != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = reinterpret_cast<PFN_encodeTiled>(f);
  return fn;
}

int g_num_sms = 0;

}  // namespace

cudaError_t make_tmap_a(CUtensorMap* m, const void* base, int C, int W, int H, int N, long long sW,
                        long long sH, long long sN, int TW, int TH, bool bf16) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return cudaErrorNotSupported;
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)sW * 2, (cuuint64_t)sH * 2, (cuuint64_t)sN * 2};
  cuuint32_t box[4] = {(cuuint32_t)kBK, (cuuint32_t)TW, (cuuint32_t)TH, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(m, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4,
                   const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

cudaError_t make_tmap_b(CUtensorMap* m, const void* base, long long K, long long rows, long long Z,
                        long long sRow, long long sZ, int BN, bool bf16) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return cudaErrorNotSupported;
  cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)rows, (cuuint64_t)Z};
  cuuint64_t strides[2] = {(cuuint64_t)sRow * 2, (cuuint64_t)sZ * 2};
  cuuint32_t box[3] = {(cuuint32_t)kBK, (cuuint32_t)BN, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(m, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3,
                   const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

static int acc_tile_bytes(const IgemmParams& p) { return 128 * p.MT * p.acc_pitch * (int)sizeof(float); }

const char* igemm_finalize(IgemmParams* p) {
  if (p->MT == 0) p->MT = 1;
  if (p->npass == 0) p->npass = 1;
  if (p->npass != 1 && p->npass != 3) return "npass must be 1 or 3";
  if (p->npass == 1) { p->pass_amap[0] = 0; p->pass_bk[0] = 0; p->pass_bmap[0] = 0; }
  if (p->out_lo && (p->stats || p->res_tma || p->patch || (p->flags & IG_OUT_F32_NCHW)))
    return "the high-precision output layout excludes epilogue statistics, TMA residuals, the patch loop and fp32 maps";
  if (p->MT != 1 && p->MT != 2) return "MT must be 1 or 2";
  if (p->BN != 16 && p->BN != 32 && p->BN != 64 && p->BN != 128) return "BN must be 16, 32, 64 or 128";
  if (p->MT == 2 && p->BN > 64) return "MT=2 needs BN <= 64 (the consumer holds at most 128 x 128 accumulators per warpgroup)";
  if (p->TW * p->TH != kBM * p->MT) return "TW*TH must be 128*MT";
  if (p->TW > 256 || p->TH > 256) return "TMA box dims are limited to 256";
  if ((1 << p->tw_shift) != p->TW) return "TW must be a power of two";
  if (p->Z0 < 1 || p->Z1 < 1) return "bad batch dims";
  p->tiles_x = (p->gridW + p->TW - 1) / p->TW;
  p->tiles_y = (p->gridH + p->TH - 1) / p->TH;
  p->n_tiles_n = (p->Cout + p->BN - 1) / p->BN;
  const int ncls = p->cls_from_z0 ? p->Z0 : 1;
  if (ncls > kMaxClasses) return "too many classes";
  for (int c = 0; c < ncls; ++c) {
    if (p->nseg[c] < 1 || p->nseg[c] > kMaxSegs) return "bad segment count";
    int n = 0;
    for (int s = 0; s < p->nseg[c]; ++s) n += p->seg[c][s].nchunks;
    p->nkb[c] = n;
    if (n < 1) return "empty K loop";
  }
  long long total = (long long)p->n_tiles_n * p->tiles_x * p->tiles_y * p->Z0 * p->Z1;
  if (total > 0x7fffffffLL) return "too many tiles";
  p->total_tiles = (int)total;
  const int stats_bytes = p->stats ? (kEpiWarps * p->Cout * 2 + kEpiWarps * 8) * (int)sizeof(float) : 0;   // epilogue_staged
  if (p->tma_store && ((p->Cout % 64) || (p->BN % 64) || (p->flags & (IG_OUT_F32_NCHW | IG_GEGLU)) || p->out_z0 != 0))
    return "staged epilogue needs Cout % 64 == 0, BN % 64 == 0, plain 16-bit NHWC output, no GEGLU";
  if (p->stats && (!p->tma_store || p->Cout > 512)) return "statistics need the staged epilogue and Cout <= 512";
  // The patch kernel at BN = 128 hands its tile over in two 64-column halves (igemm_common.cuh): a whole 128 x 128 fp32 tile
  // (64 KiB) next to the two 30 KiB halo patches and the statistics scratch would cost two of the six weight stages.
  p->acc_half = (p->patch && p->BN == 128) ? 1 : 0;
  if (p->acc_half && (!p->tma_store || p->MT != 1))
    return "patch mode at BN = 128 needs the staged epilogue and MT = 1";
  p->acc_pitch = p->acc_half ? 64 : (p->BN + 31) & ~31;
  // fixed part: staging (one 4 KiB tile per epilogue warp, x2 for the (hi, lo) layout), the accumulator tile (or half-tile),
  // 3 KiB for barriers and one N tile of bias, the statistics scratch
  const int fixed = (p->tma_store ? kEpiWarps * 4096 * (p->out_lo ? 2 : 1) : 0) + acc_tile_bytes(*p) + 3072 + stats_bytes;
  const int ring_unit = p->patch ? p->BN * 128 : kABytes * p->MT + p->BN * 128;   // bytes per pipeline stage
  if (p->patch) {
    // nine taps of the main source (map 0), then at most two 1x1 shortcut segments (maps 1, 2: the patch-box views)
    bool table = p->nseg[0] >= 9 && p->nseg[0] <= 11;
    int sc_chunks = 0;
    for (int s = 0; table && s < p->nseg[0]; ++s) {
      const IgemmSeg& sg = p->seg[0][s];
      if (s < 9) table = sg.map == 0 && sg.nchunks == p->kc_count && sg.dy == s / 3 - 1 && sg.dx == s % 3 - 1;
      else table = sg.map == s - 8 && sg.dy == 0 && sg.dx == 0;
      if (s >= 9) sc_chunks += sg.nchunks;
    }
    if (p->TW != kPatchTW || p->TH != 8 * p->MT || p->tw_shift != 4 || p->Z0 != 1 || p->Z1 < 1 || !table || p->kc_count < 1 ||
        p->nkb[0] != 9 * p->kc_count + sc_chunks || p->npass != 1 || p->gridW % p->TW || p->gridH % p->TH || !p->tma_store)
      return "patch mode needs 16 x 8 MT tiles that divide the output, a 3x3 tap table of one source (+ up to two 1x1 "
             "shortcut sources) and the staged epilogue";
    p->a_slot_bytes = (kPatchPitch * (p->TH + 2) * 128 + 1023) & ~1023;
  }
  const int avail = kMaxSmem - 1024 - fixed - (p->patch ? 2 * p->a_slot_bytes : 0);
  int st = avail / ring_unit;
  // bias: one N tile (288 floats, inside the 3 KiB) or, when the layer has several N tiles, the whole padded vector (<= 16 KiB),
  // loaded once instead of on every change of tile column, unless that costs a pipeline stage
  p->bias_slots = kBiasSlots;
  p->bias_all = 0;
  if (p->n_tiles_n > 1 && p->n_tiles_n * p->BN + 32 <= 4096) {
    const int extra = (p->n_tiles_n * p->BN + 32 - kBiasSlots) * (int)sizeof(float);
    if ((avail - extra) / ring_unit == st) {
      p->bias_all = 1;
      p->bias_slots = p->n_tiles_n * p->BN + 32;
    }
  }
  if (st > 8) st = 8;
  if (st < 2) return "tile too large for shared memory";
  p->stages = st;
  return nullptr;
}

// Function attributes are per device: keyed by the current device so that engines on several GPUs of one process work.
static cudaError_t igemm_init() {
  static bool attr_set[64] = {};
  static int sms[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
  if (!attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(igemm_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem);
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(igemm_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem);
    if (e != cudaSuccess) return e;
    cudaDeviceGetAttribute(&sms[dev], cudaDevAttrMultiProcessorCount, dev);
    attr_set[dev] = true;
  }
  g_num_sms = sms[dev];
  return cudaSuccess;
}

cudaError_t igemm_launch(const IgemmParams& p, cudaStream_t stream) {
  cudaError_t ie = igemm_init();
  if (ie != cudaSuccess) return ie;
  if (p.total_tiles <= 0) return cudaSuccess;
  if (p.stats && p.stats_slots < (p.total_tiles < g_num_sms ? p.total_tiles : g_num_sms)) return cudaErrorInvalidValue;
  const int grid = p.total_tiles < g_num_sms ? p.total_tiles : g_num_sms;
  // always request the maximum so exactly one CTA is resident per SM
  const size_t smem = kMaxSmem;
  if (p.patch) return igemm_patch_launch(p, grid, stream);
  if (p.flags & IG_BF16) {
    launch(igemm_kernel<true>, grid, kRoleThreads, smem, stream, p);
  } else {
    launch(igemm_kernel<false>, grid, kRoleThreads, smem, stream, p);
  }
  return cudaGetLastError();
}

}  // namespace gp
