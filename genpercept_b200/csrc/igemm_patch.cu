// Patch-resident wgmma implicit GEMM for 3x3 stride-1 convolutions over wide images (W % 128 == 0), with the
// producer-side GroupNorm(+SiLU) applied to the operand ON ITS WAY to the tensor core.
//
// Per 64-channel K chunk ONE (TH+2) x 130 pixel halo patch of the source lands in shared memory (a single TMA box,
// image borders zero-filled) and all nine filter taps are fed from it by row-offset SWIZZLE_128B descriptors: tap
// (dy,dx) of image row h starts ((h+dy+1)*130 + dx+1) rows into the patch (any 128-byte row is a valid descriptor
// start because the swizzle is a function of the absolute shared-memory address).
// Activation traffic L2 -> SM drops from 9 to (TH+2)*130 / (TH*128) reads per element.
//
// GroupNorm fusion (SURVEY.md §7 step 3, App. C.8; reference call sites: every `norm1 -> SiLU -> conv1` /
// `norm2 -> SiLU -> conv2` / `conv_norm_out -> SiLU -> conv_out` of the diffusers VAE blocks that
// genpercept/genpercept_pipeline.py:500,521 of the reference drive): the statistics of the source tensor come from
// its producer's epilogue (gn_finalize turns them into one (scale, shift) pair per (image, channel)); the consumer
// warpgroup rewrites each landed patch in place, y = silu(x * scale + shift), leaving the zero-filled halo pixels
// outside the image at zero (the convolution pads the NORMALISED tensor with zeros), and only then runs its wgmmas on
// it.  The normalised tensor never exists in HBM: one 2-byte read + one 2-byte write per element and one kernel launch
// less per GroupNorm.
//
// Extra K chunks for a fused 1x1 shortcut (ResnetBlock2D.conv_shortcut over the RAW block input): centre tap only,
// loaded through a second tensor map and passed through the transform untouched.
//
// Warp roles (384 threads, 1 CTA / SM, persistent; see igemm_common.cuh): warps 0..3 epilogue, warps 4..7 the wgmma
// consumer (and, with XFORM, the operand transform), warp 8 patch producer (two patch slots), warp 11 weight producer
// (one TMA box per (chunk, tap)).
#include "igemm_common.cuh"
#include "launch.h"

namespace gp {

namespace {

constexpr int kPW = kBM + 2;      // patch width in pixels (TW = 128)
constexpr int kPP = kPW;          // patch row pitch in pixels (one TMA box per patch: rows are contiguous)

__device__ __forceinline__ float silu_tanh(float x) {   // x * sigmoid(x) = h + h * tanh(h), h = x / 2 (kernels.cu silu_f)
  const float h = 0.5f * x;
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(h));
  return fmaf(h, t, h);
}
// Two channels per special-function op (tanh.approx.f16x2 has the same ~2^-11 relative error as the f32 form; h and the
// final h + h * tanh(h) stay in fp32).
__device__ __forceinline__ uint32_t silu_pair_f16(float ha, float hb) {     // inputs are already x / 2
  const __half2 h2 = __floats2half2_rn(ha, hb);
  uint32_t hi = *reinterpret_cast<const uint32_t*>(&h2), ti;
  asm("tanh.approx.f16x2 %0, %1;" : "=r"(ti) : "r"(hi));
  const float2 t = __half22float2(*reinterpret_cast<const __half2*>(&ti));
  const __half2 y = __floats2half2_rn(fmaf(ha, t.x, ha), fmaf(hb, t.y, hb));
  return *reinterpret_cast<const uint32_t*>(&y);
}

// y = silu(x * scale + shift) in place over the landed patch of chunk kc, by the 128 threads of the consumer warpgroup.
template <bool BF16>
__device__ __forceinline__ void transform_patch(const IgemmParams& p, uint32_t slot_addr, const TileCoord& t, int kc, int tt) {
  const int cpos = tt & 7;                         // 16-byte position inside the 128-byte row
  const int rbase = tt >> 3;                       // rows rbase, rbase + 16, ...
  // SWIZZLE_128B: position = logical 16-byte chunk ^ (row & 7); rows advance by 16, so (row & 7) is fixed per thread
  const int jlog = cpos ^ (rbase & 7);             // this thread's logical channel group (8 channels) in every chunk
  const bool do_silu = p.gn_silu != 0;
  const int prows = (p.TH + 2) * kPP;
  const int x0 = t.tx * p.TW - 1, y0 = t.ty * p.TH - 1;
  float sc[8], sh[8];
  const float4* sp = reinterpret_cast<const float4*>(p.gn_ss + (long long)t.z1 * p.gn_C * 2 + (kc * kBK + jlog * 8) * 2);
  const float pre = (do_silu && !BF16) ? 0.5f : 1.f;   // the fp16 SiLU form takes h = x / 2: folded into the affine
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float4 a = __ldg(sp + e);
    sc[2 * e] = a.x * pre; sh[2 * e] = a.y * pre; sc[2 * e + 1] = a.z * pre; sh[2 * e + 1] = a.w * pre;
  }
  const uint32_t base = slot_addr + cpos * 16;
  int py = 0, px = rbase;                          // rbase < 16 < kPW
  for (int r = rbase; r < prows; r += 64) {        // four rows in flight per thread
    uint32_t w[4][4];
    bool ok[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int rr = r + 16 * u;
      ok[u] = rr < prows && px < kPW && (unsigned)(y0 + py) < (unsigned)p.gridH && (unsigned)(x0 + px) < (unsigned)p.gridW;
      if (ok[u])
        asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                     : "=r"(w[u][0]), "=r"(w[u][1]), "=r"(w[u][2]), "=r"(w[u][3]) : "r"(base + rr * 128));
      px += 16;
      if (px >= kPP) { px -= kPP; ++py; }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (!ok[u]) continue;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float a = fmaf(cvt16<BF16>((uint16_t)(w[u][e] & 0xFFFF)), sc[2 * e], sh[2 * e]);
        float b = fmaf(cvt16<BF16>((uint16_t)(w[u][e] >> 16)), sc[2 * e + 1], sh[2 * e + 1]);
        if (BF16) {
          if (do_silu) { a = silu_tanh(a); b = silu_tanh(b); }
          w[u][e] = pack16<BF16>(a, b);
        } else {
          w[u][e] = do_silu ? silu_pair_f16(a, b) : pack16<BF16>(a, b);
        }
      }
      asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(base + (r + 16 * u) * 128), "r"(w[u][0]),
                   "r"(w[u][1]), "r"(w[u][2]), "r"(w[u][3]) : "memory");
    }
  }
  fence_proxy_async_shared();                      // generic-proxy writes -> visible to the tensor core's reads
  asm volatile("bar.sync 2, 128;" ::: "memory");   // the whole patch is transformed before any wgmma reads it
}

// K loop of the patch kernel for one (BN, MB = 2 * MT) instance; the whole consumer warpgroup runs it.
// One batch (the wgmmas of one (chunk, tap)) stays in flight, as in the tap kernel: after batch i is committed and batch
// i - 1 has retired, batch i - 1's weight stage is released, and so is its patch slot when it was the last batch of its
// chunk.  The weight ring holds >= 2 stages and there are two patch slots, so nothing waited for is still held.
// With XFORM, chunk kc + 1's patch is transformed while chunk kc's last batch is in flight: the two read and write
// different slots, and the slot being transformed was last read by chunk kc - 1, whose batches have all retired (its slot
// was released only after that, and the producer refilled it only after the release).  The transform's
// fence.proxy.async + bar.sync 2 still order its stores before the first wgmma that reads them.
// BN = 128: the tile goes to the epilogue in two 64-column halves (acc_half, igemm_common.cuh).
template <bool BF16, bool XFORM, int BN, int MB>
__device__ __forceinline__ void patch_consumer(const IgemmParams& p, uint8_t* smem, uint8_t* sB, float* accs, uint64_t* a_full,
                                               uint64_t* a_empty, uint64_t* b_full, uint64_t* b_empty, uint64_t* tfull_bar,
                                               uint64_t* tempty_bar, int wc, int lane) {
  float d[MB][BN / 2];
  const int b_bytes = BN * 128;
  const int kc_all = p.kc_count + p.kc_sc;
  int slot = 0, stage = 0;
  uint32_t a_phase = 0, b_phase = 0, acc_phase = 0;
  // m64 block mb covers image row mb / 2 of the tile, pixels 64 (mb & 1) ..
  auto row_off = [&](int mb, int dy, int dx) { return ((dy + 1 + (mb >> 1)) * kPP + dx + 1 + (mb & 1) * 64) * 128; };
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    const TileCoord t = decode_tile(p, tile);
    int held_stage = -1;     // weight stage of the batch in flight
    int held_slot = -1;      // patch slot whose last batch is the one in flight
    for (int kc = 0; kc < kc_all; ++kc) {
      const bool main = kc < p.kc_count;
      mbar_wait(&a_full[slot], a_phase, 3);                                                   // the patch has landed
      const uint32_t patch = smem_u32(smem + slot * p.a_slot_bytes);
      if constexpr (XFORM) {
        if (main) transform_patch<BF16>(p, patch, t, kc, wc * 32 + lane);
      }
      const int ntap = main ? 9 : 1;
      for (int tap = 0; tap < ntap; ++tap) {
        const int dy = main ? p.seg[0][tap].dy : 0, dx = main ? p.seg[0][tap].dx : 0;   // shortcut chunk: centre tap only
        mbar_wait(&b_full[stage], b_phase, 6);
        const uint64_t b_desc = make_sw128_kmajor_desc(smem_u32(sB + stage * b_bytes));
#pragma unroll
        for (int mb = 0; mb < MB; ++mb) reg_fence(d[mb]);
        wgmma_fence();
#pragma unroll
        for (int mb = 0; mb < MB; ++mb) {
          const uint64_t a_desc = make_sw128_kmajor_desc(patch + row_off(mb, dy, dx));
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

// XFORM = false: the consumer waits for the landed patch and runs its wgmmas.  XFORM = true: GroupNorm(+SiLU) of the
// patch in place first (the GroupNorm-fused build).
template <bool BF16, bool XFORM>
__global__ void __launch_bounds__(kRoleThreads, 1) igemm_patch_kernel(const __grid_constant__ IgemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int b_bytes = p.BN * 128;
  const int stages = p.stages;                       // depth of the weight ring
  uint8_t* sB = smem + 2 * p.a_slot_bytes;
  uint8_t* stg_base = sB + stages * b_bytes;
  float* accs = reinterpret_cast<float*>(stg_base + (p.tma_store ? kEpiWarps * 4096 : 0));
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
  const int kc_all = p.kc_count + p.kc_sc;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.tmPatch);
    tma_prefetch_desc(&p.tmPatch2);
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
      if (p.tma_store) run_epilogue_staged<BF16, true>(p, stg_base, sacc, sbias, tfull_bar, tempty_bar, res_bar, accs, warp, lane);
      else epilogue_direct<BF16, false>(p, sbias, tfull_bar, tempty_bar, accs, warp, lane);
    } else {
      // ===================================================================== wgmma consumer
      const int wc = warp - kConsumerWarp0;
#define GP_PATCH(BN_, MB_) patch_consumer<BF16, XFORM, BN_, MB_>(p, smem, sB, accs, a_full, a_empty, b_full, b_empty, tfull_bar, tempty_bar, wc, lane)
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
    int slot = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const TileCoord t = decode_tile(p, tile);
      const int x0 = t.tx * p.TW - 1, y0 = t.ty * p.TH - 1;
      for (int kc = 0; kc < kc_all; ++kc) {
        const bool main = kc < p.kc_count;
        mbar_wait(&a_empty[slot], phase ^ 1, 1);
        if (leader) {
          mbar_expect_tx(&a_full[slot], (uint32_t)((p.TH + 2) * kPW * 128));
          tma_load_4d(smem + slot * p.a_slot_bytes, main ? &p.tmPatch : &p.tmPatch2, &a_full[slot],
                      (main ? kc : kc - p.kc_count) * kBK, x0, y0, t.z1);
        }
        __syncwarp();
        if (++slot == 2) { slot = 0; phase ^= 1; }
      }
    }
  } else if (warp == 11) {
    // ===================================================================== weight producer
    const bool leader = elect_one();
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const TileCoord t = decode_tile(p, tile);
      const int b_row = t.n_tile * p.BN;
      for (int kc = 0; kc < kc_all; ++kc) {
        const bool main = kc < p.kc_count;
        const int ntap = main ? 9 : 1;
        for (int tap = 0; tap < ntap; ++tap) {
          // packed weights: [tap][main chunk] ... then the shortcut chunks
          const int kblk = main ? tap * p.kc_count + kc : 9 * p.kc_count + (kc - p.kc_count);
          mbar_wait(&b_empty[stage], phase ^ 1, 5);
          if (leader) {
            mbar_expect_tx(&b_full[stage], (uint32_t)b_bytes);
            tma_load_3d(sB + stage * b_bytes, &p.tmB, &b_full[stage], kblk * kBK, b_row, 0);
          }
          __syncwarp();
          if (++stage == stages) { stage = 0; phase ^= 1; }
        }
      }
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
    const void* fns[4] = {(const void*)igemm_patch_kernel<false, false>, (const void*)igemm_patch_kernel<false, true>,
                          (const void*)igemm_patch_kernel<true, false>, (const void*)igemm_patch_kernel<true, true>};
    for (const void* f : fns) {
      cudaError_t e = cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem);
      if (e != cudaSuccess) return e;
    }
    attr_set[dev] = true;
  }
  const bool xform = p.gn_ss != nullptr;
  if (p.flags & IG_BF16) {
    if (xform) launch(igemm_patch_kernel<true, true>, grid, kRoleThreads, kMaxSmem, stream, p);
    else launch(igemm_patch_kernel<true, false>, grid, kRoleThreads, kMaxSmem, stream, p);
  } else {
    if (xform) launch(igemm_patch_kernel<false, true>, grid, kRoleThreads, kMaxSmem, stream, p);
    else launch(igemm_patch_kernel<false, false>, grid, kRoleThreads, kMaxSmem, stream, p);
  }
  return cudaGetLastError();
}

}  // namespace gp
