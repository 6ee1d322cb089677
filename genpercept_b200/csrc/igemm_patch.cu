// Patch-resident wgmma implicit GEMM for 3x3 stride-1 convolutions whose 16 x 8 MT pixel tiles divide the output.
//
// The M tile is built from 8 x 8-pixel m64 blocks: TW = 16 (two blocks across) by TH = 8 MT (MT blocks down).  Per
// 64-channel K chunk ONE (TH+2) x kPatchPitch pixel halo patch of the source lands in shared memory (a single TMA box,
// image borders zero-filled, the columns past TW + 2 over-fetched and never read) and all nine filter taps are fed from it
// by row-offset SWIZZLE_128B descriptors: core group g (pixel row g) of block (bx, by) for tap (dy, dx) starts at patch row
// (8 by + g + dy + 1) * kPatchPitch + 8 bx + dx + 1, and the groups are kPatchPitch * 128 bytes apart (a multiple of 1024,
// so every group has the swizzle phase of the first; any 128-byte row is a valid start because the swizzle is a function
// of the absolute shared-memory address).  Activation traffic L2 -> SM drops from 9 to 10 * 24 / 128 = 1.9 (MT = 1) or
// 18 * 24 / 256 = 1.7 (MT = 2) reads per element.
// A fused 1x1 shortcut (ResNets that change the channel count) is more K chunks: after the nine-tap loop over the main
// source, each shortcut chunk is loaded through the same patch slots with the same box and feeds the centre tap only; its
// weights follow the nine taps in the packed matrix.
//
// Warp roles (384 threads, 1 CTA / SM, persistent; see igemm_common.cuh): warps 0..3 the staged epilogue, warps 4..7 the
// wgmma consumer, warp 8 patch producer (two patch slots), warp 11 weight producer (one TMA box per (chunk, tap)).
#include "igemm_common.cuh"
#include "launch.h"

namespace gp {

namespace {

constexpr uint32_t kGroupStride = kPatchPitch * 128;   // bytes between the 8-row core groups of an m64 block

// 64-channel K chunks of the shortcut sources (segments 9.. of the tap table, one per source)
__device__ __forceinline__ int shortcut_chunks(const IgemmParams& p) {
  int n = 0;
  for (int s = 9; s < p.nseg[0]; ++s) n += p.seg[0][s].nchunks;
  return n;
}

// K loop of the patch kernel for one (BN, MB = 2 * MT) instance; the whole consumer warpgroup runs it.
// One batch (the wgmmas of one (chunk, tap)) stays in flight, as in the tap kernel: after batch i is committed and batch
// i - 1 has retired, batch i - 1's weight stage is released, and so is its patch slot when it was the last batch of its
// chunk.  The weight ring holds >= 2 stages and there are two patch slots, so nothing waited for is still held.
// BN = 128: the tile goes to the epilogue in two 64-column halves (acc_half, igemm_common.cuh).
template <bool BF16, int BN, int MB>
__device__ __forceinline__ void patch_consumer(const IgemmParams& p, uint8_t* smem, uint8_t* sB, float* accs, uint64_t* a_full,
                                               uint64_t* a_empty, uint64_t* b_full, uint64_t* b_empty, uint64_t* tfull_bar,
                                               uint64_t* tempty_bar, int wc, int lane) {
  float d[MB][BN / 2];
  const int b_bytes = BN * 128;
  const int nchunks = p.kc_count + shortcut_chunks(p);
  int slot = 0, stage = 0;
  uint32_t a_phase = 0, b_phase = 0, acc_phase = 0;
  // m64 block mb is the 8 x 8 pixels (bx, by) = (mb & 1, mb >> 1) of the tile; its first row, tap (dy, dx)
  auto row_off = [&](int mb, int dy, int dx) { return ((8 * (mb >> 1) + dy + 1) * kPatchPitch + 8 * (mb & 1) + dx + 1) * 128; };
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    int held_stage = -1;     // weight stage of the batch in flight
    int held_slot = -1;      // patch slot whose last batch is the one in flight
    for (int kc = 0; kc < nchunks; ++kc) {
      mbar_wait(&a_full[slot], a_phase, 3);                                                   // the patch has landed
      const uint32_t patch = smem_u32(smem + slot * p.a_slot_bytes);
      const int ntap = kc < p.kc_count ? 9 : 1;                                               // shortcut chunks: centre tap
      for (int tap = 0; tap < ntap; ++tap) {
        const int dy = ntap == 9 ? p.seg[0][tap].dy : 0, dx = ntap == 9 ? p.seg[0][tap].dx : 0;
        mbar_wait(&b_full[stage], b_phase, 6);
        const uint64_t b_desc = make_sw128_kmajor_desc(smem_u32(sB + stage * b_bytes));
#pragma unroll
        for (int mb = 0; mb < MB; ++mb) reg_fence(d[mb]);
        wgmma_fence();
#pragma unroll
        for (int mb = 0; mb < MB; ++mb) {
          const uint64_t a_desc = make_sw128_kmajor_desc(patch + row_off(mb, dy, dx), kGroupStride);
#pragma unroll
          for (int k = 0; k < kBK / 16; ++k) wgmma_ss<BN, BF16>(d[mb], a_desc + 2 * k, b_desc + 2 * k, (kc | tap | k) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();                            // the previous batch has retired
#pragma unroll
        for (int mb = 0; mb < MB; ++mb) reg_fence(d[mb]);
        if (held_stage >= 0) {
          __syncwarp();
          if (lane == 0) {
            mbar_arrive(&b_empty[held_stage]);
            if (held_slot >= 0) mbar_arrive(&a_empty[held_slot]);
          }
          held_slot = -1;
        }
        held_stage = stage;
        if (++stage == p.stages) { stage = 0; b_phase ^= 1; }
      }
      held_slot = slot;
      if (++slot == 2) { slot = 0; a_phase ^= 1; }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int mb = 0; mb < MB; ++mb) reg_fence(d[mb]);
    __syncwarp();
    if (lane == 0) {
      mbar_arrive(&b_empty[held_stage]);
      mbar_arrive(&a_empty[held_slot]);
    }
    if constexpr (BN == 128) {                   // two 64-column halves through the 64-column shared tile
      mbar_wait(tempty_bar, acc_phase ^ 1, 2);
      acc_store<BN, MB, 0, 8>(accs, p.acc_pitch, d, wc, lane);
      mbar_arrive(tfull_bar);
      acc_phase ^= 1;
      mbar_wait(tempty_bar, acc_phase ^ 1, 2);
      acc_store<BN, MB, 8, 8>(accs, p.acc_pitch, d, wc, lane);
      mbar_arrive(tfull_bar);
      acc_phase ^= 1;
    } else {
      mbar_wait(tempty_bar, acc_phase ^ 1, 2);   // the epilogue has read the previous tile
      acc_store<BN, MB>(accs, p.acc_pitch, d, wc, lane);
      mbar_arrive(tfull_bar);
      acc_phase ^= 1;
    }
  }
}

template <bool BF16>
__global__ void __launch_bounds__(kRoleThreads, 1) igemm_patch_kernel(const __grid_constant__ IgemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int b_bytes = p.BN * 128;
  const int stages = p.stages;                       // depth of the weight ring
  uint8_t* sB = smem + 2 * p.a_slot_bytes;
  uint8_t* stg_base = sB + stages * b_bytes;         // one 4 KiB staging tile per epilogue warp
  float* accs = reinterpret_cast<float*>(stg_base + kEpiWarps * 4096);
  uint64_t* a_full = reinterpret_cast<uint64_t*>(accs + 128 * p.MT * p.acc_pitch);   // [slot]
  uint64_t* a_empty = a_full + 2;
  uint64_t* b_full = a_empty + 2;
  uint64_t* b_empty = b_full + stages;
  uint64_t* tfull_bar = b_empty + stages;
  uint64_t* tempty_bar = tfull_bar + 1;
  uint64_t* res_bar = tempty_bar + 1;                                  // [epilogue warps] residual tile landed
  float* sbias = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(res_bar + kEpiWarps) + 15) & ~uintptr_t(15));   // [bias_slots]
  float* sacc = sbias + p.bias_slots;

  const int warp = uniform_warp_id();
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.tmPatch);
    for (int s = 9; s < p.nseg[0]; ++s) tma_prefetch_desc(&p.tmA[p.seg[0][s].map]);
    tma_prefetch_desc(&p.tmB);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&a_full[i], 1);
      mbar_init(&a_empty[i], 4);                     // the four consumer warps
    }
    for (int i = 0; i < stages; ++i) { mbar_init(&b_full[i], 1); mbar_init(&b_empty[i], 4); }
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
    if (warp < kEpiWarps) {
      // ===================================================================== epilogue
      run_epilogue_staged<BF16, true>(p, stg_base, sacc, sbias, tfull_bar, tempty_bar, res_bar, accs, warp, lane);
    } else {
      // ===================================================================== wgmma consumer
      const int wc = warp - kConsumerWarp0;
#define GP_PATCH(BN_, MB_) patch_consumer<BF16, BN_, MB_>(p, smem, sB, accs, a_full, a_empty, b_full, b_empty, tfull_bar, tempty_bar, wc, lane)
      if (p.MT == 2) {
        if (p.BN == 16) GP_PATCH(16, 4); else if (p.BN == 32) GP_PATCH(32, 4); else GP_PATCH(64, 4);
      } else {
        if (p.BN == 16) GP_PATCH(16, 2); else if (p.BN == 32) GP_PATCH(32, 2); else if (p.BN == 64) GP_PATCH(64, 2); else GP_PATCH(128, 2);
      }
#undef GP_PATCH
    }
    return;
  }
  setmaxnreg_dec<kProducerRegs>();
  if (warp == 8) {
    // ===================================================================== patch producer
    const bool leader = elect_one();
    const uint32_t patch_bytes = (uint32_t)((p.TH + 2) * kPatchPitch * 128);
    int slot = 0;
    uint32_t phase = 0;
    auto load = [&](const CUtensorMap* tm, int k0, int x0, int y0, int z) {
      mbar_wait(&a_empty[slot], phase ^ 1, 1);
      if (leader) {
        mbar_expect_tx(&a_full[slot], patch_bytes);
        tma_load_4d(smem + slot * p.a_slot_bytes, tm, &a_full[slot], k0, x0, y0, z);
      }
      __syncwarp();
      if (++slot == 2) { slot = 0; phase ^= 1; }
    };
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const TileCoord t = decode_tile(p, tile);
      const int x0 = t.tx * p.TW - 1, y0 = t.ty * p.TH - 1;
      for (int kc = 0; kc < p.kc_count; ++kc) load(&p.tmPatch, kc * kBK, x0, y0, t.z1);
      for (int s = 9; s < p.nseg[0]; ++s)                                     // shortcut sources
        for (int c = 0; c < p.seg[0][s].nchunks; ++c) load(&p.tmA[p.seg[0][s].map], c * kBK, x0, y0, t.z1);
    }
  } else if (warp == 11) {
    // ===================================================================== weight producer
    const bool leader = elect_one();
    const int nsc = shortcut_chunks(p);
    int stage = 0;
    uint32_t phase = 0;
    auto load = [&](int kblk, int b_row) {
      mbar_wait(&b_empty[stage], phase ^ 1, 5);
      if (leader) {
        mbar_expect_tx(&b_full[stage], (uint32_t)b_bytes);
        tma_load_3d(sB + stage * b_bytes, &p.tmB, &b_full[stage], kblk * kBK, b_row, 0);
      }
      __syncwarp();
      if (++stage == stages) { stage = 0; phase ^= 1; }
    };
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const TileCoord t = decode_tile(p, tile);
      const int b_row = t.n_tile * p.BN;
      for (int kc = 0; kc < p.kc_count; ++kc) {
        // kept rolled: unrolled nine times, the default bench.py step ran about 0.2 % slower on an H100 80GB HBM3 (700 W)
#pragma unroll 1
        for (int tap = 0; tap < 9; ++tap) load(tap * p.kc_count + kc, b_row);   // packed weights: [tap][chunk]
      }
      for (int i = 0; i < nsc; ++i) load(9 * p.kc_count + i, b_row);            // then the shortcut segments
    }
  }
}

}  // namespace

cudaError_t igemm_patch_launch(const IgemmParams& p, int grid, cudaStream_t stream) {
  static bool attr_set[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
  if (!attr_set[dev]) {
    for (const void* f : {(const void*)igemm_patch_kernel<false>, (const void*)igemm_patch_kernel<true>}) {
      cudaError_t e = cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem);
      if (e != cudaSuccess) return e;
    }
    attr_set[dev] = true;
  }
  if (p.flags & IG_BF16) launch(igemm_patch_kernel<true>, grid, kRoleThreads, kMaxSmem, stream, p);
  else launch(igemm_patch_kernel<false>, grid, kRoleThreads, kMaxSmem, stream, p);
  return cudaGetLastError();
}

}  // namespace gp
