// Plan-time arena and op-list builder: turns layer-level calls (conv, attention, norms ...) into
// fully parameterised kernel launches (tensor maps encoded once, at plan time).
#include <algorithm>
#include <cmath>
#include <cstring>

#include "engine.h"
#include "fattn.h"
#include "fattn512.h"

namespace gp {

// Single-head d = 512 attention (the VAE mid-block) takes the fused kernel (fattn512.cu) once the unfused path's score
// matrix S would exceed this many bytes, or where the unfused path cannot run at all (rows longer than softmax_rows
// takes).  Below it the unfused path (QK^T GEMM -> softmax -> P V GEMM) is kept: it is what every size up to and
// including bench.py's largest configuration (8 x 768^2: 1.36 GB of S) has always run, so those outputs stay
// bit-identical.  Above it S alone decides whether a photo fits on the card (49 GB at 2592 x 3872), while the fused
// kernel needs no workspace at all.
constexpr size_t kFusedAttnMinBytes = size_t(2) << 30;

// ------------------------------------------------------------------------------------ Arena
size_t Arena::alloc(size_t bytes) {
  bytes = (bytes + 1023) & ~size_t(1023);
  if (bytes == 0) bytes = 1024;
  for (size_t i = 0; i < blks_.size(); ++i) {
    if (blks_[i].free && blks_[i].size >= bytes) {
      if (blks_[i].size > bytes) {
        Blk rest{blks_[i].off + bytes, blks_[i].size - bytes, true};
        blks_[i].size = bytes;
        blks_.insert(blks_.begin() + i + 1, rest);
      }
      blks_[i].free = false;
      return blks_[i].off;
    }
  }
  size_t off = blks_.empty() ? 0 : blks_.back().off + blks_.back().size;
  if (!blks_.empty() && blks_.back().free) {   // grow the trailing free block
    off = blks_.back().off;
    blks_.back().size = bytes;
    blks_.back().free = false;
  } else {
    blks_.push_back(Blk{off, bytes, false});
  }
  high_ = std::max(high_, off + bytes);
  return off;
}

void Arena::release(size_t off) {
  for (size_t i = 0; i < blks_.size(); ++i) {
    if (blks_[i].off == off && !blks_[i].free) {
      blks_[i].free = true;
      if (i + 1 < blks_.size() && blks_[i + 1].free) {
        blks_[i].size += blks_[i + 1].size;
        blks_.erase(blks_.begin() + i + 1);
      }
      if (i > 0 && blks_[i - 1].free) {
        blks_[i - 1].size += blks_[i].size;
        blks_.erase(blks_.begin() + i);
      }
      return;
    }
  }
  throw GpError(GP_ERR_STATE, "arena: release of unknown block");
}

// ------------------------------------------------------------------------------------ Builder
Builder::Builder(bool bf16, bool measuring, uint8_t* base, bool split)
    : bf16_(bf16), measuring_(measuring), split_(split), base_(base) {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
    num_sms = n;
}
T4 Builder::alloc(int N, int H, int W, int C) {
  T4 t;
  t.N = N; t.H = H; t.W = W; t.C = C;
  t.planes = split_ ? 2 : 1;
  t.off = (long long)arena_.alloc(t.bytes());
  return t;
}
T4 Builder::external(const void* p, int N, int H, int W, int C) const {
  T4 t;
  t.N = N; t.H = H; t.W = W; t.C = C;
  t.planes = split_ ? 2 : 1;
  t.off = (long long)(reinterpret_cast<const uint8_t*>(p) - base_);
  return t;
}
void Builder::release(const T4& t) {
  auto it = stats.find(t.off);
  if (it != stats.end()) {
    arena_.release(it->second.off);
    stats.erase(it);
  }
  arena_.release((size_t)t.off);
}

void Builder::push(const std::string& name, int launches, double flops, double bytes,
                   std::function<cudaError_t(cudaStream_t)> fn) {
  Op o;
  o.name = name;
  o.stage = stage;
  o.variant = variant;
  o.launches = launches;
  o.flops = flops;
  o.bytes = bytes;
  o.run = std::move(fn);
  ops.push_back(std::move(o));
}
void Builder::custom(const std::string& name, int launches, double bytes, std::function<cudaError_t(cudaStream_t)> fn) {
  if (measuring_) return;
  push(name, launches, 0, bytes, std::move(fn));
}

// N tile: one of the wgmma widths the GEMM kernels are built for (16, 32, 64, 128).  Cout = 320 (the SD-2.1 UNet's first
// level) takes 64 (five exact tiles): a multiple of 64 keeps the staged TMA-store epilogue.
int choose_bn(int cout, int force) {
  if (force) return force;
  for (int bn : {16, 32, 64})
    if (cout <= bn) return bn;
  return (cout % 128 == 0 || cout % 64 != 0) ? 128 : 64;
}
// pick the TW x TH = `rows` (128 or 256) patch with the least padding waste (ties: wider rows)
static void choose_tile(int gw, int gh, int rows, int* tw, int* th, int* shift) {
  double best = 1e30;
  for (int s = 7; s >= 0; --s) {
    const int w = 1 << s, h = rows >> s;
    if (h > 256) continue;
    const double waste = (double)ceil_div(gw, w) * w * ceil_div(gh, h) * h / ((double)gw * gh);
    if (waste < best - 1e-9) { best = waste; *tw = w; *th = h; *shift = s; }
  }
}

// Tile shape (BN, MT) for the layers that do not fill the GPU (the UNet's deep levels at any batch, everything at batch
// 1).  Two bounds per candidate: the tensor time of the longest-running SM — ceil(tiles / SMs) waves of tiles whose
// duration scales with the MMA width (a narrow MMA is bound by its operand fetch) — and the L2 -> SM operand traffic,
// tiles x K x (128 MT + BN) x 2 bytes.  A candidate replaces the default only for a predicted gain above 10 %, so every
// layer with many waves stays where choose_bn put it.
struct TileShape { int bn, mt; };
template <class MTilesFn>
static TileShape choose_tile_shape(int cout, double k_elems, int num_sms, TileShape dflt, MTilesFn mtiles_of) {
  if (cout % 64 != 0 || cout < 128) return dflt;
  auto cost = [&](TileShape t) {
    const double tiles = (double)mtiles_of(t.mt) * ceil_div(cout, t.bn);
    const double waves = std::ceil(tiles / num_sms);
    const double cyc_per_kb = 4.0 * t.mt * (t.bn == 64 ? 48.0 : t.bn / 2.0);
    const double t_mma = waves * ((k_elems / 64.0) * cyc_per_kb / 1.5e9 + 3e-6);     // + epilogue / pipeline fill per wave
    const double t_l2 = tiles * k_elems * (128.0 * t.mt + t.bn) * 2.0 / 7.0e12;
    return std::max(t_mma, t_l2);
  };
  TileShape best = dflt;
  const double c0 = cost(dflt);
  double best_cost = c0;
  for (int bn : {128, 64})
    for (int mt : {1, 2}) {
      if (mt == 2 && bn > 64) continue;
      const double c = cost(TileShape{bn, mt});
      if (c < 0.9 * c0 && c < best_cost) { best_cost = c; best = TileShape{bn, mt}; }
    }
  return best;
}
// Default (choose_bn, two M tiles when the N tile is narrow and the layer fills the GPU) + the model above, for a stride-1
// layer of `images` maps of gw x gh output pixels (tokens_mode: one row of images * gw * gh tokens).  Host-only; exported
// as gp_tile_shape so that the decision table is pinned by a CPU test.
void tile_shape_for(int cout, double k_elems, bool tokens_mode, int images, int gw, int gh, int num_sms, int* bn, int* mt) {
  const long long work_px = (long long)images * gw * gh;
  const int bn0 = choose_bn(cout, 0);
  const int mt0 = (bn0 <= 64 && work_px >= 256LL * num_sms) ? 2 : 1;
  auto mtiles_of = [&](int m) -> long long {
    if (tokens_mode) return (work_px + 128 * m - 1) / (128 * m);
    int tw = 128, th = m, sh = 7;
    choose_tile(gw, gh, 128 * m, &tw, &th, &sh);
    return (long long)images * ceil_div(gw, tw) * ceil_div(gh, th);
  };
  const TileShape ts = choose_tile_shape(cout, k_elems, num_sms, TileShape{bn0, mt0}, mtiles_of);
  *bn = ts.bn;
  *mt = ts.mt;
}

// Whether a 3x3 stride-1 layer's planned (BN, MT) tile runs on the patch-resident kernel as far as its shape goes: the
// 16 x 8 MT pixel tile (igemm_patch.cu) divides the output exactly, there are at least as many tiles as SMs, and a shortcut
// is no wider than the main source.  Ragged edges and the small maps stay on the tap-streaming kernel.  (The caller checks the rest: mode 0, 3x3, the staged
// epilogue, one main source plus at most two shortcut sources, not the high-precision mode.)
// A fused 1x1 shortcut (csc channels over a cin-channel main source) is taken along only while it is no wider than the main
// source: each shortcut chunk loads a whole halo patch for one batch of MMAs, and with two patch slots those loads are no
// longer hidden.  On an H100 80GB HBM3 (700 W) the VAE's 256 + 128 and 512 + 256 shortcut layers ran 6 % and 26 % faster
// on the patch kernel, while 256 + 512, 128 + 256 and the UNet's up-block layers (shortcut 1.5-3x the main source) ran
// up to 26 % slower than on the tap-streaming kernel.
bool patch_tile_fits(int images, int h, int w, int cin, int csc, int cout, int bn, int mt, int num_sms) {
  const int th = 8 * mt;
  if (w % kPatchTW || h % th || csc > cin) return false;
  return (long long)images * (w / kPatchTW) * (h / th) * ceil_div(cout, bn) >= num_sms;
}

static void check_cuda(cudaError_t e, const std::string& what) {
  if (e != cudaSuccess) throw GpError(GP_ERR_CUDA, what + ": " + cudaGetErrorString(e));
}
static void finalize_or_throw(IgemmParams* p, const std::string& name) {
  const char* err = igemm_finalize(p);
  if (err) throw GpError(GP_ERR_INVALID, name + ": " + err);
}

// A operand view `slot` of box (64, p.TW, p.TH); in the high-precision mode also its lo plane, `lo` elements further
// with the same strides, as view slot + 4
void Builder::tmap_a(IgemmParams& p, int slot, const void* base, long long lo, int C, int W, int H, int N, long long sW,
                     long long sH, long long sN, const std::string& what) const {
  check_cuda(make_tmap_a(&p.tmA[slot], base, C, W, H, N, sW, sH, sN, p.TW, p.TH, bf16_), what);
  if (split_)
    check_cuda(make_tmap_a(&p.tmA[slot + 4], reinterpret_cast<const uint16_t*>(base) + lo, C, W, H, N, sW, sH, sN, p.TW, p.TH,
                           bf16_), what + " lo");
}
// An activation B operand of box (64, p.BN, 1) in tmB; in the high-precision mode its lo plane, `lo` elements further, in
// tmB2.  (Packed weights carry their lo plane along K: one tmB.)
void Builder::tmap_b(IgemmParams& p, const void* base, long long lo, long long K, long long rows, long long Z, long long sRow,
                     long long sZ, const std::string& what) const {
  check_cuda(make_tmap_b(&p.tmB, base, K, rows, Z, sRow, sZ, p.BN, bf16_), what);
  if (split_)
    check_cuda(make_tmap_b(&p.tmB2, reinterpret_cast<const uint16_t*>(base) + lo, K, rows, Z, sRow, sZ, p.BN, bf16_), what + " lo");
}
// The A views past the first `used` repeat view 0 (and their lo planes view 4)
static void fill_a_slots(IgemmParams& p, int used) {
  for (int i = used; i < 4; ++i) {
    p.tmA[i] = p.tmA[0];
    p.tmA[i + 4] = p.tmA[4];
  }
}
// The high-precision mode's three GEMM passes: hi*hi + lo*hi + hi*lo (A planes at tmA[0..3] / tmA[4..7]).  B's lo plane
// follows its hi plane along K at `b_lo_k` (packed weights) or, with b_lo_k = 0, is tmB2.  `out_lo`: IgemmParams::out_lo.
static void set_passes(IgemmParams& p, int b_lo_k, long long out_lo) {
  p.npass = 3;
  p.pass_amap[0] = 0; p.pass_amap[1] = 4; p.pass_amap[2] = 0;
  p.pass_bk[0] = 0; p.pass_bk[1] = 0; p.pass_bk[2] = b_lo_k;
  p.pass_bmap[0] = 0; p.pass_bmap[1] = 0; p.pass_bmap[2] = b_lo_k ? 0 : 1;
  p.out_lo = out_lo;
}
// A batched GEMM over one row of M tokens per batch index (the attention GEMMs and to_vT): 128 x 1 M tiles, one K segment
// of `kchunks` 64-channel chunks, the N tile for `cout` columns.  The caller sets the batch coordinates, output and operands.
static void token_gemm(IgemmParams& p, bool bf16, int M, int cout, int kchunks) {
  std::memset(&p, 0, sizeof(p));
  p.flags = bf16 ? IG_BF16 : 0;
  p.gridW = M; p.gridH = 1; p.TW = 128; p.TH = 1; p.tw_shift = 7;
  p.nseg[0] = 1;
  p.seg[0][0] = IgemmSeg{0, 0, 0, (uint16_t)kchunks};
  p.outW = M; p.outH = 1;
  p.out_row_stride = 0;
  p.out_sy = p.out_sx = 1;
  p.Cout = cout;
  p.BN = choose_bn(cout, 0);
}
void Builder::push_igemm(const std::string& name, IgemmParams& p, double flops, double bytes) {
  finalize_or_throw(&p, name);
  push(name, 1, flops, bytes, [p](cudaStream_t s) { return igemm_launch(p, s); });
  ops.back().kind = 1;
}

void Builder::conv(const std::string& name, const ConvArgs& a) {
  GP_REQUIRE(!a.srcs.empty() && a.w != nullptr, name + ": bad conv args");
  if (a.gn != nullptr) {      // materialise GroupNorm(+SiLU)(concat(srcs)), then the plain convolution
    int ctot = 0;
    for (auto& s : a.srcs) ctot += s.C;
    T4 tmp = alloc(a.srcs[0].N, a.srcs[0].H, a.srcs[0].W, ctot);
    gn(a.gn_name, a.srcs, *a.gn, a.gn_groups, a.gn_eps, a.gn_silu, tmp);
    ConvArgs b = a;
    b.gn = nullptr;
    b.srcs = {tmp};
    conv(name, b);
    release(tmp);
    return;
  }
  const T4& s0 = a.srcs[0];
  const int N = s0.N, H = s0.H, W = s0.W;
  const auto [Ho, Wo] = conv_out_dims(a.mode, H, W);
  const int PL = split_ ? 2 : 1;
  const int out_cl = a.out_f32 ? 0 : a.out.C;   // logical channels of the 16-bit output ...
  const int out_c = out_cl * PL;                // ... and its pixel stride in elements
  GP_REQUIRE(a.w->planes == PL, name + ": packed weights do not match the engine's precision mode");
  if (split_) {   // a source's lo plane starts C elements into the pixel: a TMA base must be 16-byte aligned
    for (auto& s : a.srcs) GP_REQUIRE(s.C % 8 == 0, name + ": the (hi, lo) layout needs source channels % 8 == 0");
    for (auto& s : a.sc) GP_REQUIRE(s.C % 8 == 0, name + ": the (hi, lo) layout needs shortcut channels % 8 == 0");
    GP_REQUIRE(!(a.flags & IG_GEGLU) || out_cl % 8 == 0, name + ": the (hi, lo) GEGLU output needs channels % 8 == 0");
  }
  const int Cout = a.cout_valid > 0 ? a.cout_valid : a.out.C;
  int cin_total = 0;
  for (auto& s : a.srcs) cin_total += s.C;
  double flops = 2.0 * N * Ho * Wo * (double)Cout * cin_total * a.ks * a.ks;
  for (auto& s : a.sc) flops += 2.0 * N * Ho * Wo * (double)Cout * s.C;
  double bytes = (double)N * Ho * Wo * Cout * (a.out_f32 ? 4 : 2) + (double)a.w->rows * a.w->ktot * a.w->nz * 2;
  for (auto& s : a.srcs) bytes += (double)s.bytes();
  for (auto& s : a.sc) bytes += (double)s.bytes();
  if (a.res1) bytes += (double)a.res1->bytes();
  if (a.res2) bytes += (double)a.res2->bytes();
  if (!a.out_f32) GP_REQUIRE(a.out.N == N && a.out.H == Ho && a.out.W == Wo, name + ": output shape mismatch");
  // GroupNorm partial sums from the epilogue: same decision (and arena allocation) in both passes
  const bool tokens_mode = (a.ks == 1 && a.mode == 0 && a.sc.empty() && a.srcs.size() == 1 && !a.out_f32);
  const long long ntok = (long long)N * H * W;
  // extent of the tile grid: the output, or in mode 3 the input grid of each of the four parity classes
  const int gw = a.mode == 3 ? W : Wo, gh = a.mode == 3 ? H : Ho;
  const long long work_px = tokens_mode ? ntok : (long long)gw * gh * N * (a.mode == 3 ? 4 : 1);
  int bn_pre = choose_bn(Cout, a.force_bn);
  int mt_pre = (bn_pre <= 64 && work_px >= 256LL * num_sms) ? 2 : 1;
  if (!a.force_bn && !(a.flags & IG_GEGLU)) {
    const double k_elems = flops / (2.0 * N * Ho * Wo * (double)Cout) * (a.mode == 3 ? 4.0 / 9.0 : 1.0);
    tile_shape_for(Cout, k_elems, tokens_mode, N * (a.mode == 3 ? 4 : 1), gw, gh, num_sms, &bn_pre, &mt_pre);
  }
  // the staged (TMA store) epilogue wherever the output allows it; GEGLU and fp32 maps take the direct epilogue
  const bool staged = !a.out_f32 && !(a.flags & IG_GEGLU) && Cout == a.out.C && (Cout % 64) == 0 && (bn_pre % 64) == 0;
  // The patch-resident kernel keeps the planned (BN, MT).  At BN = 128 it hands the accumulators over in two 64-column
  // halves through a 32 KiB tile, so with the two 30 KiB halo patches six 16 KiB weight stages fit next to the statistics
  // scratch of any Cout <= 512.
  int csc = 0;
  for (auto& s : a.sc) csc += s.C;
  const bool patch_eligible = staged && a.mode == 0 && a.ks == 3 && a.srcs.size() == 1 && a.sc.size() <= 2 && !split_ &&
                              patch_tile_fits(N, Ho, Wo, s0.C, csc, Cout, bn_pre, mt_pre, num_sms);
  bool emit_stats = a.want_stats && staged && Cout <= 512 && !split_;
  if (emit_stats && tokens_mode && ((long long)H * W) % (128 * mt_pre) != 0) emit_stats = false;
  size_t stats_off = 0;
  const size_t stats_bytes = (size_t)N * num_sms * Cout * kGnRec * sizeof(float);
  if (emit_stats) {
    GP_REQUIRE(stats.find(a.out.off) == stats.end(), name + ": output already has statistics");
    stats_off = arena_.alloc(stats_bytes);
    stats[a.out.off] = StatsInfo{stats_off, num_sms, Cout};
  }
  if (measuring_) return;

  IgemmParams p;
  std::memset(&p, 0, sizeof(p));
  p.flags = a.flags | (bf16_ ? IG_BF16 : 0) | (a.out_f32 ? IG_OUT_F32_NCHW : 0);
  p.bias = a.w->bias;
  p.res1 = a.res1 ? ptr(*a.res1) : nullptr;
  p.res2 = a.res2 ? ptr(*a.res2) : nullptr;
  p.out = a.out_f32 ? (void*)a.out_f32 : ptr(a.out);
  p.Cout = Cout;
  p.BN = bn_pre;
  p.Z1 = 1; p.Z0 = 1;
  p.out_sy = p.out_sx = 1;
  int nmap = 0;   // A views in use
  if (tokens_mode) {
    GP_REQUIRE(ntok < (1LL << 31), name + ": too many tokens");
    p.gridW = (int)ntok; p.gridH = 1;
    p.MT = mt_pre;
    p.TW = 128 * p.MT; p.TH = 1; p.tw_shift = p.MT == 2 ? 8 : 7;
    p.nseg[0] = 1;
    p.seg[0][0] = IgemmSeg{0, 0, 0, (uint16_t)ceil_div(s0.C, 64)};
    p.outW = (int)ntok; p.outH = 1;
    p.out_pix_stride = out_c; p.out_row_stride = 0;
    tmap_a(p, nmap++, ptr(s0), s0.C, s0.C, (int)ntok, 1, 1, s0.ps(), ntok * s0.ps(), ntok * s0.ps(), name + ": tmap A");
  } else {
    p.Z1 = N;
    p.a_n_z1 = 1;
    p.outW = Wo; p.outH = Ho;
    p.out_pix_stride = out_c;
    p.out_row_stride = (long long)Wo * out_c;
    p.out_z1 = (long long)Ho * Wo * out_c;
    p.gridW = gw;
    p.gridH = gh;
    // two accumulator tiles per CTA when the N tile is narrow and there is enough work to fill the GPU
    p.MT = mt_pre;
    if (patch_eligible) { p.TW = kPatchTW; p.TH = 8 * p.MT; p.tw_shift = 4; }
    else choose_tile(p.gridW, p.gridH, 128 * p.MT, &p.TW, &p.TH, &p.tw_shift);
    if (a.mode == 0 || a.mode == 3) {
      GP_REQUIRE(a.srcs.size() + a.sc.size() <= 4, name + ": too many sources");
      auto add_src = [&](const T4& s) {
        tmap_a(p, nmap++, ptr(s), s.C, s.C, W, H, N, s.ps(), (long long)W * s.ps(), (long long)H * W * s.ps(), name + ": tmap A");
      };
      for (auto& s : a.srcs) {
        GP_REQUIRE(s.N == N && s.H == H && s.W == W, name + ": source shape mismatch");
        add_src(s);
      }
      for (auto& s : a.sc) {
        GP_REQUIRE(s.N == N && s.H == H && s.W == W && a.mode == 0, name + ": shortcut shape mismatch");
        add_src(s);
      }
    } else {
      GP_REQUIRE(a.srcs.size() == 1 && a.sc.empty() && H >= 2 && W >= 2, name + ": stride-2 needs one source");
      for (int hp = 0; hp < 2; ++hp)
        for (int wp = 0; wp < 2; ++wp) {
          const uint8_t* b = reinterpret_cast<const uint8_t*>(ptr(s0)) + ((long long)hp * W + wp) * s0.ps() * 2;
          tmap_a(p, hp * 2 + wp, b, s0.C, s0.C, (W - wp + 1) / 2, (H - hp + 1) / 2, N, 2LL * s0.ps(), 2LL * W * s0.ps(),
                 (long long)H * W * s0.ps(), name + ": tmap A");
        }
      nmap = 4;
    }
    if (a.mode == 0) {
      int ns = 0;
      const int half = a.ks / 2;
      for (int r = 0; r < a.ks; ++r)
        for (int s = 0; s < a.ks; ++s)
          for (size_t i = 0; i < a.srcs.size(); ++i)
            p.seg[0][ns++] = IgemmSeg{(int8_t)i, (int8_t)(r - half), (int8_t)(s - half), (uint16_t)ceil_div(a.srcs[i].C, 64)};
      for (size_t j = 0; j < a.sc.size(); ++j)
        p.seg[0][ns++] = IgemmSeg{(int8_t)(a.srcs.size() + j), 0, 0, (uint16_t)ceil_div(a.sc[j].C, 64)};
      GP_REQUIRE(ns <= kMaxSegs, name + ": too many K segments");
      p.nseg[0] = ns;
    } else if (a.mode == 1 || a.mode == 2) {
      const int pad = (a.mode == 1) ? 1 : 0;
      int ns = 0;
      for (int r = 0; r < 3; ++r)
        for (int s = 0; s < 3; ++s) {
          const int ty = r - pad, tx = s - pad;
          const int hp = ((ty % 2) + 2) % 2, wp = ((tx % 2) + 2) % 2;
          p.seg[0][ns++] = IgemmSeg{(int8_t)(hp * 2 + wp), (int8_t)((ty - hp) / 2), (int8_t)((tx - wp) / 2),
                                    (uint16_t)ceil_div(s0.C, 64)};
        }
      p.nseg[0] = ns;
    } else {
      p.Z0 = 4;
      p.cls_from_z0 = 1;
      p.b_z_z0 = 1;
      p.out_sy = p.out_sx = 2;
      for (int c = 0; c < 4; ++c) {
        const int py = c >> 1, px = c & 1;
        p.cls_py[c] = (int8_t)py; p.cls_px[c] = (int8_t)px;
        int ns = 0;
        for (int aa = 0; aa < 2; ++aa)
          for (int bb = 0; bb < 2; ++bb)
            p.seg[c][ns++] = IgemmSeg{0, (int8_t)(py - 1 + aa), (int8_t)(px - 1 + bb), (uint16_t)ceil_div(s0.C, 64)};
        p.nseg[c] = ns;
      }
    }
  }
  fill_a_slots(p, nmap);
  check_cuda(make_tmap_b(&p.tmB, a.w->w, (long long)a.w->ktot * PL, a.w->rows, a.w->nz, (long long)a.w->ktot * PL,
                         (long long)a.w->rows * a.w->ktot * PL, p.BN, bf16_), name + ": tmap B");
  if (split_) set_passes(p, a.w->ktot, out_cl);   // the weights' lo plane follows the hi plane along K
  if (staged) {   // output tensor maps for the TMA-store epilogue (one per parity class)
    p.tma_store = 1;
    // a warp stores 32 tile rows: min(TW, 32) x (32 / that) pixels, or an 8 x 4 piece of an m64 block of a patch tile
    const int bw = patch_eligible ? 8 : p.TW < 32 ? p.TW : 32, bh = 32 / bw;
    // maps of out_cl channels at the output's pixel stride over `base`, in the output's geometry
    auto epilogue_maps = [&](CUtensorMap* m, const uint8_t* base, const std::string& what) {
      if (a.mode == 3) {
        for (int c = 0; c < 4; ++c) {
          const int py = c >> 1, px = c & 1;
          const uint8_t* ob = base + ((long long)py * Wo + px) * out_c * 2;
          check_cuda(make_tmap_a(&m[c], ob, out_cl, W, H, N, 2LL * out_c, 2LL * Wo * out_c, (long long)Ho * Wo * out_c, bw, bh,
                                 bf16_), what);
        }
        return;
      }
      if (tokens_mode)
        check_cuda(make_tmap_a(&m[0], base, out_cl, (int)ntok, 1, 1, out_c, ntok * out_c, ntok * out_c, bw, bh, bf16_), what);
      else
        check_cuda(make_tmap_a(&m[0], base, out_cl, Wo, Ho, N, out_c, (long long)Wo * out_c, (long long)Ho * Wo * out_c,
                               bw, bh, bf16_), what);
      for (int i = 1; i < 4; ++i) m[i] = m[0];
    };
    for (int pl = 0; pl < PL; ++pl)           // plane 0: tmOut, plane 1 (high-precision lo): tmOutLo
      epilogue_maps(pl == 0 ? p.tmOut : p.tmOutLo, reinterpret_cast<const uint8_t*>(ptr(a.out)) + (size_t)pl * out_cl * 2,
                    name + ": tmap out");
    // the residual has the output's shape and addressing: same maps over its base (one plane: out_c == out_cl)
    if (a.res1 && !a.res2 && !split_) {
      p.res_tma = 1;
      epilogue_maps(p.tmRes, reinterpret_cast<const uint8_t*>(ptr(*a.res1)), name + ": tmap res");
    }
  }
  // patch-resident main loop: the main source and the shortcut sources (tmA[1..2]) as halo-patch boxes
  if (patch_eligible) {
    p.patch = 1;
    p.kc_count = ceil_div(s0.C, 64);
    auto patch_map = [&](CUtensorMap* m, const T4& s) {
      check_cuda(make_tmap_a(m, ptr(s), s.C, W, H, N, s.ps(), (long long)W * s.ps(), (long long)H * W * s.ps(), kPatchPitch,
                             p.TH + 2, bf16_), name + ": tmap patch");
    };
    patch_map(&p.tmPatch, s0);
    for (size_t j = 0; j < a.sc.size(); ++j) patch_map(&p.tmA[1 + j], a.sc[j]);
  }
  if (emit_stats) {
    p.stats = reinterpret_cast<float*>(raw_ptr(stats_off));
    p.stats_slots = num_sms;
    p.stats_hw = tokens_mode ? H * W : 0;
  }
  finalize_or_throw(&p, name);
  GP_REQUIRE(p.MT == mt_pre && p.BN == bn_pre, name + ": tile pre-selection disagrees with the plan");
  const int ncls = p.cls_from_z0 ? p.Z0 : 1;
  for (int c = 0; c < ncls; ++c)
    GP_REQUIRE(p.nkb[c] * 64 == a.w->ktot, name + ": packed K (" + std::to_string(a.w->ktot) + ") != planned K (" +
                                              std::to_string(p.nkb[c] * 64) + ")");
  GP_REQUIRE(a.w->rows >= Cout, name + ": packed rows < Cout");
  if (emit_stats) {
    float* sp = p.stats;
    push(name, 2, flops, bytes, [p, sp, stats_bytes](cudaStream_t s) {
      cudaError_t e = cudaMemsetAsync(sp, 0, stats_bytes, s);
      if (e != cudaSuccess) return e;
      return igemm_launch(p, s);
    });
  } else if (a.out_f32 && out_slot) {
    float** slot = out_slot;
    push(name, 1, flops, bytes, [p, slot](cudaStream_t s) {
      IgemmParams q = p;
      q.out = *slot;
      return igemm_launch(q, s);
    });
  } else {
    push(name, 1, flops, bytes, [p](cudaStream_t s) { return igemm_launch(p, s); });
  }
  ops.back().kind = 1;
  if (a.mode == 3) ops.back().flops_exec = flops * 4.0 / 9.0;      // four 2x2 parity convs instead of a 3x3 on the 2x grid
}

void Builder::attention_qkv(const std::string& name, const void* q, const void* k, long long cs, const void* vT, int B,
                            int T, int heads, int d, const float* pv_bias, const T4& out, long long qk_lo) {
  // High-precision mode: q / k carry their lo planes `qk_lo` elements further (same pixel stride cs), V^T rows are
  // [hi Tp | lo Tp], S / P rows likewise; the three GEMM passes of IgemmParams::npass do hi*hi + lo*hi + hi*lo.
  const int Tp = ceil_div(T, 8) * 8;
  const int C = heads * d;
  const int PL = split_ ? 2 : 1;
  const long long TpP = (long long)Tp * PL;   // physical row pitch of S and V^T
  // The high-precision mode takes the fused kernels only when memory-efficient attention is switched on; by default
  // its plans store S.
  const bool split_fused = split_ && mem_efficient_attn;
  // the fused kernels' params (FattnParams / Fattn512Params) but for `heads` / `bias`: Q and K boxes of q_box tokens, and
  // in the high-precision mode the lo planes' maps
  auto fattn_setup = [&](auto& p, int q_box) {
    std::memset(&p, 0, sizeof(p));
    p.out = ptr(out);
    p.out_b_stride = (long long)T * out.ps();
    p.out_row_stride = (int)out.ps();
    p.T = T; p.B = B; p.q_tiles = ceil_div(T, q_box);
    p.scale_log2e = 1.4426950408889634f;
    p.bf16 = bf16_ ? 1 : 0;
    check_cuda(make_tmap_b(&p.tmQ, q, C, T, B, cs, (long long)T * cs, q_box, bf16_), name + ": tmap Q");
    check_cuda(make_tmap_b(&p.tmK, k, C, T, B, cs, (long long)T * cs, q_box, bf16_), name + ": tmap K");
    check_cuda(make_tmap_b(&p.tmV, vT, T, C, B, TpP, (long long)C * TpP, 64, bf16_), name + ": tmap Vt");
    if (!split_) return;
    const uint16_t* ql = reinterpret_cast<const uint16_t*>(q) + qk_lo;
    const uint16_t* kl = reinterpret_cast<const uint16_t*>(k) + qk_lo;
    const uint16_t* vl = reinterpret_cast<const uint16_t*>(vT) + Tp;
    check_cuda(make_tmap_b(&p.tmQl, ql, C, T, B, cs, (long long)T * cs, q_box, false), name + ": tmap Q lo");
    check_cuda(make_tmap_b(&p.tmKl, kl, C, T, B, cs, (long long)T * cs, q_box, false), name + ": tmap K lo");
    check_cuda(make_tmap_b(&p.tmVl, vl, T, C, B, TpP, (long long)C * TpP, 64, false), name + ": tmap Vt lo");
    p.split = 1;
    p.out_lo = out.C;
  };
  if (d == 64 && (!split_ || split_fused)) {   // fused wgmma flash-attention kernel (S and P stay on chip)
    if (measuring_) return;
    FattnParams p;
    fattn_setup(p, 128);
    p.heads = heads;
    push(name + ".fattn", 1, 4.0 * B * heads * (double)T * T * d, 4.0 * B * T * C * 2 * PL,
         [p](cudaStream_t s) { return fattn_launch(p, s); });
    ops.back().kind = 2;
    return;
  }
  const size_t s_bytes = (size_t)B * heads * T * TpP * 2;
  // the unfused path's softmax_rows cannot take rows past kSoftmaxRowsMaxT keys when T is a multiple of 8
  const bool unfused_runs = T % 8 != 0 || T <= kSoftmaxRowsMaxT;
  const bool fused512 = d == 512 && heads == 1 &&
                        (split_ ? split_fused
                                : attn512_path >= 0 ? attn512_path == 1 : s_bytes > kFusedAttnMinBytes || !unfused_runs);
  if (fused512) {   // fused d = 512 kernel: no score matrix in the arena
    if (measuring_) return;
    Fattn512Params p;
    fattn_setup(p, 64);
    p.bias = pv_bias;
    push(name + ".fattn512", 1, 4.0 * B * (double)T * T * d, 4.0 * B * T * C * 2 * PL,
         [p](cudaStream_t s) { return fattn512_launch(p, s); });
    ops.back().kind = 2;
    return;
  }
  if (!unfused_runs && long_softmax.empty()) long_softmax = name;
  const size_t s_off = arena_.alloc(s_bytes);
  if (!measuring_) {
    void* S = raw_ptr(s_off);
    {  // S = Q K^T  (softmax scale is folded into Wq)
      IgemmParams p;
      token_gemm(p, bf16_, T, T, ceil_div(d, 64));
      p.Z1 = B; p.Z0 = heads;
      p.a_n_z1 = 1; p.a_k_z0 = d;
      p.b_z_z1 = 1; p.b_k_z0 = d;
      p.out = S;
      p.out_pix_stride = TpP;
      p.out_z1 = (long long)heads * T * TpP; p.out_z0 = (long long)T * TpP;
      tmap_a(p, 0, q, qk_lo, C, T, 1, B, cs, (long long)T * cs, (long long)T * cs, name + ": tmap Q");
      fill_a_slots(p, 1);
      tmap_b(p, k, qk_lo, C, T, B, cs, (long long)T * cs, name + ": tmap K");
      if (split_) set_passes(p, 0, Tp);
      push_igemm(name + ".qk", p, 2.0 * B * heads * (double)T * T * d, (double)s_bytes + 2.0 * B * T * C * 2);
    }
    {
      const long long rows = (long long)B * heads * T;
      const bool bf = bf16_;
      const bool sp = split_;
      push(name + ".softmax", 1, 0, 2.0 * s_bytes, [S, rows, T, Tp, bf, sp](cudaStream_t s) { return softmax_rows(S, rows, T, Tp, bf, s, sp); });
    }
    {  // O = P V
      IgemmParams p;
      token_gemm(p, bf16_, T, d, ceil_div(T, 64));
      p.Z1 = B; p.Z0 = heads;
      p.a_n_z1 = heads; p.a_n_z0 = 1;
      p.b_z_z1 = 1; p.b_row_z0 = d;
      p.out = ptr(out);
      p.out_pix_stride = out.ps();
      p.out_z1 = (long long)T * out.ps(); p.out_z0 = d;
      p.bias = pv_bias;
      tmap_a(p, 0, S, Tp, T, T, 1, B * heads, TpP, (long long)T * TpP, (long long)T * TpP, name + ": tmap P");
      fill_a_slots(p, 1);
      tmap_b(p, vT, Tp, T, C, B, TpP, (long long)C * TpP, name + ": tmap Vt");
      if (split_) set_passes(p, 0, out.C);
      push_igemm(name + ".pv", p, 2.0 * B * heads * (double)T * T * d, (double)s_bytes + 2.0 * B * T * C * 2);
    }
  }
  arena_.release(s_off);
}

void Builder::attention(const std::string& name, const T4& l, const PackedW& wqk, const PackedW& wv,
                        const float* pv_bias, int heads, const T4& out) {
  const int B = l.N, T = l.H * l.W, C = l.C, d = C / heads;
  const int Tp = ceil_div(T, 8) * 8;
  T4 qk = alloc(B, l.H, l.W, 2 * C);
  {
    ConvArgs a;
    a.srcs = {l}; a.ks = 1; a.w = &wqk; a.out = qk;
    conv(name + ".to_qk", a);
  }
  const int PL = split_ ? 2 : 1;
  const long long TpP = (long long)Tp * PL;
  GP_REQUIRE(wv.planes == PL && wqk.planes == PL, name + ": packed weights do not match the engine's precision mode");
  const size_t vt_off = arena_.alloc((size_t)B * C * TpP * 2);
  to_vT(name, l, wv, measuring_ ? nullptr : raw_ptr(vt_off));
  const uint16_t* qp = measuring_ ? nullptr : reinterpret_cast<const uint16_t*>(ptr(qk));
  attention_qkv(name, qp, qp ? qp + C : nullptr, qk.ps(), measuring_ ? nullptr : raw_ptr(vt_off), B, T, heads, d, pv_bias, out,
                split_ ? 2LL * C : 0);
  arena_.release(vt_off);
  release(qk);
}

void Builder::to_vT(const std::string& name, const T4& l, const PackedW& wv, void* vT) {
  if (measuring_) return;
  // V^T[b] = Wv . l[b]^T : A = weights (rows = channels), B = tokens
  const int B = l.N, T = l.H * l.W, C = l.C;
  const int Tp = ceil_div(T, 8) * 8;
  const int PL = split_ ? 2 : 1;
  const long long TpP = (long long)Tp * PL;
  const size_t vt_bytes = (size_t)B * C * TpP * 2;
  IgemmParams p;
  token_gemm(p, bf16_, C, T, wv.ktot / 64);
  p.Z1 = B; p.Z0 = 1;
  p.b_z_z1 = 1;
  p.out = vT;
  p.out_pix_stride = TpP;
  p.out_z1 = (long long)C * TpP;
  const long long wrow = (long long)wv.ktot * PL;
  tmap_a(p, 0, wv.w, wv.ktot, wv.ktot, C, 1, 1, wrow, (long long)C * wrow, (long long)C * wrow, name + ": tmap Wv");
  fill_a_slots(p, 1);
  tmap_b(p, ptr(l), C, C, T, B, l.ps(), (long long)T * l.ps(), name + ": tmap l");
  if (split_) set_passes(p, 0, Tp);
  push_igemm(name + ".to_vT", p, 2.0 * B * (double)T * C * C, (double)vt_bytes + (double)l.bytes());
}

// GroupNorm(+SiLU) of concat(srcs) into out.  Each source's partial sums are either already produced by the conv that
// wrote it, or computed by a gn_stats pass into a buffer of this op's own (allocated and released here, so both passes
// make the same arena allocations).  gn_finalize turns them into a scale / shift per (image, channel) in gn_ss, then one
// gn_apply pass per source writes its channels of out.
void Builder::gn(const std::string& name, const std::vector<T4>& srcs, const NormW& nw, int groups, float eps,
                 bool silu, const T4& out) {
  int ctot = 0;
  for (auto& s : srcs) ctot += s.C;
  GP_REQUIRE(ctot == out.C && nw.C == ctot && ctot % groups == 0 && srcs.size() <= 2, name + ": GroupNorm channel mismatch");
  const int N = out.N;
  const long long HW = (long long)out.H * out.W;
  const int chunks = gn_chunks(N, HW);
  int launches = 1;
  double bytes = (double)out.bytes();
  struct Pass { const void* x; float* partial; int C; };
  std::vector<Pass> passes;
  std::vector<size_t> own;
  std::vector<GnSrc> gs(srcs.size());
  for (size_t i = 0; i < srcs.size(); ++i) {
    auto it = stats.find(srcs[i].off);
    if (it != stats.end() && it->second.C == srcs[i].C) {
      gs[i] = GnSrc{measuring_ ? nullptr : reinterpret_cast<const float*>(raw_ptr(it->second.off)), it->second.slots, srcs[i].C};
    } else {
      own.push_back(arena_.alloc((size_t)N * chunks * srcs[i].C * kGnRec * sizeof(float)));
      float* partial = measuring_ ? nullptr : reinterpret_cast<float*>(raw_ptr(own.back()));
      gs[i] = GnSrc{partial, chunks, srcs[i].C};
      if (!measuring_) passes.push_back(Pass{ptr(srcs[i]), partial, srcs[i].C});
      ++launches;
      bytes += (double)srcs[i].bytes();
    }
  }
  for (size_t off : own) arena_.release(off);
  if (measuring_) return;
  std::vector<const void*> xs;
  std::vector<int> cs;
  for (auto& s : srcs) {
    xs.push_back(ptr(s));
    cs.push_back(s.C);
    bytes += (double)s.bytes();
    ++launches;
  }
  void* y = ptr(out);
  float* ss = gn_ss;
  const bool bf = bf16_, sp = split_;
  const float* gamma = nw.gamma;
  const float* beta = nw.beta;
  push(name, launches, 0, bytes, [=](cudaStream_t s) {
    for (const Pass& q : passes) {
      cudaError_t e = gn_stats(q.x, N, HW, q.C, q.partial, chunks, q.C, 0, bf, s, sp);
      if (e != cudaSuccess) return e;
    }
    cudaError_t e = gn_finalize(gs.data(), (int)gs.size(), gamma, beta, N, ctot, groups, HW, eps, ss, s);
    if (e != cudaSuccess) return e;
    int coff = 0;
    for (size_t i = 0; i < xs.size(); ++i) {
      e = gn_apply(xs[i], N, HW, cs[i], ss, ctot, coff, y, ctot, silu, bf, s, sp);
      if (e != cudaSuccess) return e;
      coff += cs[i];
    }
    return cudaSuccess;
  });
}

void Builder::ln(const std::string& name, const T4& x, const NormW& nw, float eps, const T4& out) {
  GP_REQUIRE(nw.C == x.C && out.C == x.C, name + ": LayerNorm channel mismatch");
  if (measuring_) return;
  const void* xi = ptr(x);
  void* yo = ptr(out);
  const long long tokens = x.pixels();
  const int C = x.C;
  const bool bf = bf16_;
  const float* g = nw.gamma;
  const float* b = nw.beta;
  const bool sp = split_;
  push(name, 1, 0, 2.0 * x.bytes(), [=](cudaStream_t s) { return layernorm(xi, yo, tokens, C, g, b, eps, bf, s, sp); });
}

void Builder::xattn(const std::string& name, const T4& x, const XattnW& w, float eps, const T4& out) {
  GP_REQUIRE(w.C == x.C, name + ": cross-attention channel mismatch");
  if (measuring_) return;
  const void* xi = ptr(x);
  void* yo = ptr(out);
  const long long tokens = x.pixels();
  const bool bf = bf16_, sp = split_;
  const XattnW ww = w;
  push(name, 1, 4.0 * tokens * (double)w.C * w.heads, 2.0 * x.bytes(), [=](cudaStream_t s) {
    return xattn2(xi, yo, tokens, ww.C, ww.heads, ww.U, ww.u0, ww.M, ww.c0, eps, bf, s, sp);
  });
}

void Builder::relu_op(const std::string& name, const T4& in, const T4& out) {
  if (measuring_) return;
  const void* xi = ptr(in);
  void* yo = ptr(out);
  const long long n = in.pixels() * in.C;
  const bool bf = bf16_;
  const int sc = split_ ? in.C : 0;
  push(name, 1, 0, 2.0 * in.bytes(), [=](cudaStream_t s) { return relu16(xi, yo, n, bf, s, sc); });
}

void Builder::bilinear(const std::string& name, const T4& in, const T4& out) {
  GP_REQUIRE(out.H == 2 * in.H && out.W == 2 * in.W && out.C == in.C, name + ": bilinear shape mismatch");
  if (measuring_) return;
  const void* xi = ptr(in);
  void* yo = ptr(out);
  const T4 t = in;
  const bool bf = bf16_;
  const bool sp = split_;
  push(name, 1, 0, (double)in.bytes() + out.bytes(), [=](cudaStream_t s) { return bilinear_up2x(xi, yo, t.N, t.H, t.W, t.C, bf, s, sp); });
}

void Builder::resize(const std::string& name, const T4& in, const T4& out, bool nearest) {
  GP_REQUIRE(out.N == in.N && out.C == in.C, name + ": resize shape mismatch");
  if (measuring_) return;
  const void* xi = ptr(in);
  void* yo = ptr(out);
  const int n = in.N, h = in.H, w = in.W, oh = out.H, ow = out.W, c = in.C;
  const bool bf = bf16_, sp = split_;
  const int ch = (int)in.ps();
  push(name, 1, 0, (double)in.bytes() + (double)out.bytes(), [=](cudaStream_t s) {
    return nearest ? nearest_resize(xi, yo, n, h, w, oh, ow, ch, s) : bilinear_resize(xi, yo, n, h, w, oh, ow, c, bf, s, sp);
  });
}

void Builder::direct(const std::string& name, const T4& in, int cin, const DirectW& w, const T4& out, float* out_f32) {
  GP_REQUIRE(w.Cin == cin, name + ": direct conv channel mismatch");
  if (measuring_) return;
  DirectConvParams p;
  std::memset(&p, 0, sizeof(p));
  p.in = ptr(in);
  p.N = in.N; p.H = in.H; p.W = in.W; p.Cin = cin; p.in_cstride = (int)in.ps();
  p.in_lo = split_ ? in.C : 0;
  p.w = w.w; p.bias = w.bias;
  p.Ho = in.H; p.Wo = in.W;
  p.Cout = w.Cout;
  p.ks = w.ks; p.stride = 1; p.pad = w.ks / 2;
  p.flags = out_f32 ? DC_OUT_F32_NCHW : 0;
  if (out_f32) { p.out = out_f32; p.out_cstride = w.Cout; }
  else { p.out = ptr(out); p.out_cstride = (int)out.ps(); p.out_lo = split_ ? out.C : 0; }
  const bool bf = bf16_;
  const double flops = 2.0 * p.N * p.Ho * p.Wo * (double)p.Cout * cin * w.ks * w.ks;
  float** slot = out_f32 ? out_slot : nullptr;
  push(name, 1, flops, (double)in.bytes() + (double)p.N * p.Ho * p.Wo * p.Cout * (out_f32 ? 4 : 2),
       [p, bf, slot](cudaStream_t s) {
         if (!slot) return direct_conv(p, bf, s);
         DirectConvParams q = p;
         q.out = *slot;
         return direct_conv(q, bf, s);
       });
}

}  // namespace gp
