// Internal C++ types of the engine: host weight store, packed device weights, the plan-time
// activation arena and op list builder.  The public surface is include/genpercept_b200.h.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <functional>
#include <map>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

#include "../../include/genpercept_b200.h"
#include "igemm.h"
#include "kernels.h"
#include "status.h"

namespace gp {

constexpr float kLatentScale = 0.18215f;   // genpercept_pipeline.py:96

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// Output extent (Ho, Wo) of a convolution over an H x W input in ConvArgs::mode `mode`.
inline std::pair<int, int> conv_out_dims(int mode, int H, int W) {
  if (mode == 1) return {(H + 2 - 3) / 2 + 1, (W + 2 - 3) / 2 + 1};
  if (mode == 2) return {(H + 1 - 3) / 2 + 1, (W + 1 - 3) / 2 + 1};
  if (mode == 3) return {2 * H, 2 * W};
  return {H, W};
}

// fp32 <-> 16-bit storage values (fp16, or bf16 when `bf16`), round to nearest
uint16_t host_f2h(float f, bool bf16);
float host_h2f(uint16_t u, bool bf16);

struct HostT {
  std::vector<float> d;
  std::vector<int64_t> shape;
  int64_t numel() const { int64_t n = 1; for (auto s : shape) n *= s; return n; }
};

// K-major 16-bit matrix [nz][rows][ktot] (+ fp32 bias[rows]) on the device.
struct PackedW {
  uint16_t* w = nullptr;
  int rows = 0, ktot = 0, nz = 1;
  int planes = 1;            // 2 in the high-precision mode: every row is [ktot hi | ktot lo] (value = hi + lo)
  float* bias = nullptr;
};
struct NormW { float* gamma = nullptr; float* beta = nullptr; int C = 0; };
struct XattnW { float* U = nullptr; float* u0 = nullptr; float* M = nullptr; float* c0 = nullptr; int C = 0, heads = 0; };
struct DirectW { float* w = nullptr; float* bias = nullptr; int Cin = 0, Cout = 0, ks = 0; };

// value(co, c) = sum_t coef_t * p_t[co * sco_t + c * sc_t]
struct Term { const float* p; long long sco, sc; float coef; };
struct SegSpec { std::vector<Term> terms; int C; };

// dense 16-bit NHWC activation; `off` is a byte offset into the arena (or an absolute address
// when the builder's base is null).
// High-precision mode: planes == 2, a pixel holds [hi C | lo C] (two fp16 planes, value = hi + lo).
struct T4 {
  long long off = -1;
  int N = 0, H = 0, W = 0, C = 0;
  int planes = 1;
  size_t bytes() const { return (size_t)N * H * W * C * 2 * planes; }
  long long pixels() const { return (long long)N * H * W; }
  long long ps() const { return (long long)C * planes; }      // elements between consecutive pixels
};

class Arena {
 public:
  size_t alloc(size_t bytes);
  void release(size_t off);
  size_t high_water() const { return high_; }
 private:
  struct Blk { size_t off, size; bool free; };
  std::vector<Blk> blks_;
  size_t high_ = 0;
};

struct Op {
  std::string name;
  int stage = 0;
  int variant = 0;            // 0: always; 1 / 3: only when out_channels matches
  int launches = 1;
  int kind = 0;               // 1: wgmma implicit-GEMM launch, 2: fused attention, 0: anything else
  double flops = 0, bytes = 0;   // algorithmic work (SURVEY.md 8d): what the reference's op costs
  double flops_exec = -1;        // MMA work actually issued when it differs (upsample-fused convs run 4 of 9 taps); -1: = flops
  float usec = 0;
  std::function<cudaError_t(cudaStream_t)> run;
};

struct ConvArgs {
  std::vector<T4> srcs;       // concatenated sources of the main taps
  int ks = 3;
  int mode = 0;               // 0 s1, 1 s2 pad 1, 2 s2 pad (0,1,0,1), 3 nearest-2x then s1
  std::vector<T4> sc;         // raw sources of a fused 1x1 shortcut (extra K segments)
  const PackedW* w = nullptr;
  T4 out;                     // 16-bit NHWC destination (ignored when out_f32 != null)
  int cout_valid = -1;        // columns to store (default out.C)
  const T4* res1 = nullptr;
  const T4* res2 = nullptr;
  int flags = 0;
  float* out_f32 = nullptr;   // fp32 NCHW destination [N, cout_valid, Ho, Wo]
  int force_bn = 0;
  bool want_stats = false;    // let the epilogue emit GroupNorm partial sums of `out` (consumed by Builder::gn)
  // GroupNorm(+SiLU) over concat(srcs) in front of the convolution (norm1 / norm2 / conv_norm_out of the diffusers
  // blocks).  Builder::conv materialises the normalised tensor with Builder::gn and convolves that.
  const NormW* gn = nullptr;
  std::string gn_name;
  int gn_groups = 32;
  float gn_eps = 1e-6f;
  bool gn_silu = true;
};

class Builder {
 public:
  Builder(bool bf16, bool measuring, uint8_t* base, bool split = false);
  bool split() const { return split_; }
  T4 alloc(int N, int H, int W, int C);
  T4 external(const void* p, int N, int H, int W, int C) const;
  void release(const T4& t);
  void* ptr(const T4& t) const { return base_ + t.off; }
  size_t raw_alloc(size_t bytes) { return arena_.alloc(bytes); }
  void* raw_ptr(size_t off) const { return base_ + off; }

  void conv(const std::string& name, const ConvArgs& a);
  // generic batched GEMM pieces of attention; q/k/v views live inside `qk` / `l`
  void attention(const std::string& name, const T4& l, const PackedW& wqk, const PackedW& wv, const float* pv_bias,
                 int heads, const T4& out);
  // V^T[b] = Wv . l[b]^T into vT: [B][C][Tp] with Tp = T rounded up to 8 (rows [hi Tp | lo Tp] in the high-precision mode)
  void to_vT(const std::string& name, const T4& l, const PackedW& wv, void* vT);
  void attention_qkv(const std::string& name, const void* q, const void* k, long long qk_cstride, const void* vT, int B,
                     int T, int heads, int d, const float* pv_bias, const T4& out, long long qk_lo = 0);
  void gn(const std::string& name, const std::vector<T4>& srcs, const NormW& nw, int groups, float eps, bool silu,
          const T4& out);
  void ln(const std::string& name, const T4& x, const NormW& nw, float eps, const T4& out);
  void xattn(const std::string& name, const T4& x, const XattnW& w, float eps, const T4& out);
  void relu_op(const std::string& name, const T4& in, const T4& out);
  void bilinear(const std::string& name, const T4& in, const T4& out);
  // F.interpolate(size=(out.H, out.W)) of `in`: nearest (a gather of whole pixels, both planes of the (hi, lo) layout at
  // once) or bilinear with align_corners=False
  void resize(const std::string& name, const T4& in, const T4& out, bool nearest);
  void direct(const std::string& name, const T4& in, int cin, const DirectW& w, const T4& out, float* out_f32);
  void custom(const std::string& name, int launches, double bytes, std::function<cudaError_t(cudaStream_t)> fn);

  struct StatsInfo { size_t off; int slots; int C; };
  std::map<long long, StatsInfo> stats;   // live tensors (by arena offset) whose producer emitted GN partial sums
  int num_sms = 132;   // H100 SXM; replaced by the device's count at construction

  std::vector<Op> ops;
  int stage = 0;
  int variant = 0;
  bool bf16() const { return bf16_; }
  bool measuring() const { return measuring_; }
  size_t arena_bytes() const { return arena_.high_water(); }
  float* gn_ss = nullptr;
  // When set, ops that write the final fp32 map (ConvArgs::out_f32 / direct(..., out_f32)) read their destination from
  // *out_slot at LAUNCH time, so gp_infer can point them at the caller's device buffer (no copy of the result).
  float** out_slot = nullptr;
  // Single-head d = 512 attention path: -1 chooses by the size of the score matrix (kFusedAttnMinBytes, builder.cu);
  // 0 forces the unfused path, 1 the fused kernel.  Only gp_bench_attention sets it, to time both paths at one shape.
  int attn512_path = -1;
  // High-precision mode: run every d = 64 and single-head d = 512 attention through the fused kernels, so no score matrix
  // is stored (gp_set_memory_efficient_attention).  The 16-bit modes ignore it.
  bool mem_efficient_attn = false;
  // Set when an unfused attention was planned whose softmax_rows cannot run (rows past kSoftmaxRowsMaxT keys with T a
  // multiple of 8): the name of the first such op.
  std::string long_softmax;

 private:
  void push(const std::string& name, int launches, double flops, double bytes,
            std::function<cudaError_t(cudaStream_t)> fn);
  // finalize p, push its launch, mark the op as an implicit GEMM
  void push_igemm(const std::string& name, IgemmParams& p, double flops, double bytes);
  // GEMM operand tensor maps, with the high-precision mode's lo plane `lo` elements after the hi plane (builder.cu)
  void tmap_a(IgemmParams& p, int slot, const void* base, long long lo, int C, int W, int H, int N, long long sW, long long sH,
              long long sN, const std::string& what) const;
  void tmap_b(IgemmParams& p, const void* base, long long lo, long long K, long long rows, long long Z, long long sRow,
              long long sZ, const std::string& what) const;
  bool bf16_, measuring_, split_ = false;
  uint8_t* base_;
  Arena arena_;
};

// weights.cu: the checkpoint's host tensors and the device weights packed from them (constant folding + packing,
// SURVEY.md App. C).  Every accessor packs and uploads on first use and returns the cached result afterwards, so one
// measuring pass over a topology uploads exactly the weights that topology reaches.  The store owns every device
// allocation it makes and frees them when it is destroyed.
class WeightStore {
 public:
  explicit WeightStore(bool bf16 = false, bool split = false) : bf16(bf16), split(split) {}
  ~WeightStore();
  WeightStore(const WeightStore&) = delete;
  WeightStore& operator=(const WeightStore&) = delete;

  bool bf16;
  bool split;                // cfg.precision == 1: (hi, lo) fp16 pairs everywhere (T4::planes, PackedW::planes)
  std::unordered_map<std::string, HostT> host;
  std::vector<float> text_embed;
  int n_tokens = 0;
  size_t weight_bytes = 0;
  float* pq_dev = nullptr;   // vae.post_quant_conv: [16] weight + [4] bias, fp32 on the device
  int cur_timestep = 0;      // the timestep whose biases the live conv1 bias slots hold once the queued work has run

  void put(const std::string& key, std::vector<int64_t> shape, const float* d);
  template <class Tp>
  Tp* upload(const std::vector<Tp>& v) {
    void* d = device_alloc(std::max<size_t>(v.size() * sizeof(Tp), 16));
    GP_CUDA(cudaMemcpy(d, v.data(), v.size() * sizeof(Tp), cudaMemcpyHostToDevice));
    weight_bytes += v.size() * sizeof(Tp);
    return reinterpret_cast<Tp*>(d);
  }
  void* device_alloc(size_t bytes);   // freed with the store; not counted in weight_bytes

  PackedW pack(const std::vector<std::vector<SegSpec>>& classes, int rows, const std::vector<float>& bias);
  const PackedW& conv_w(const std::string& key, const std::vector<int>& srcC, const std::string& sc_key = "",
                        const std::vector<int>& scC = {}, const std::vector<float>* extra_bias = nullptr,
                        bool want_bias = true, const std::string& cache_suffix = "");
  const PackedW& conv_up_w(const std::string& key);
  const PackedW& mat_w(const std::string& cache_key, int rows, int K, const float* m, const std::vector<float>& bias);
  const PackedW& lin_w(const std::string& key, bool bias = true);
  const NormW& norm_w(const std::string& key);
  const DirectW& direct_w(const std::string& key, int cin_used, const std::vector<float>* w_override = nullptr,
                          const std::vector<float>* b_override = nullptr, int cout_override = 0);
  const XattnW& xattn_w(const std::string& blk, int C, int heads);
  struct XattnGen { const PackedW* A; const PackedW* B; int Kp; };
  XattnGen xattn_general_w(const std::string& blk, int C, int heads);

  // folded weights of the graph (weights.cu says what each one folds)
  const PackedW& resnet_conv1(const std::string& p, int cin, bool temb_on);
  const PackedW& self_attn_qk(const std::string& blk, int C, int heads);
  const PackedW& geglu_w(const std::string& blk, int C);
  const PackedW& vae_attn_qk(const std::string& a);
  const float* vae_v_bias(const std::string& a);
  const PackedW& encoder_conv_in();
  const PackedW& encoder_tail();
  const PackedW& unet_conv_out_plain();
  const PackedW& unet_tail();
  const PackedW& decoder_tail1();
  int unet_in_channels();
  // the text tower's fused [q / 8 ; k ; v] projection of self-attention `p` (bias folded the same way), and a checkpoint
  // tensor uploaded as it is, fp32 (the embedding tables)
  const PackedW& text_qkv_w(const std::string& p);
  const float* f32_w(const std::string& key);

  void compute_temb(int timestep);
  void set_timestep(int timestep);
  // The live conv1 bias buffer (rows() floats) of time-embedded ResNet `p`, or null when `p` has none.
  float* temb_bias_slot(const std::string& p, int* rows) const;
  // The number of time-embedded ResNets packed so far.
  int temb_slot_count() const { return (int)temb_layers.size(); }
  // conv1.bias + time_emb_proj(silu(emb(timestep))) of ResNet `p`, the value set_timestep writes (cached per timestep).
  const std::vector<float>& temb_bias(int timestep, const std::string& p);

 private:
  const HostT& T(const std::string& k) const;
  bool has(const std::string& k) const { return host.count(k) != 0; }
  void upload_post_quant();
  std::vector<float> temb_for(int timestep) const;
  const std::vector<std::vector<float>>& temb_biases(int timestep);

  std::vector<void*> dev_allocs;
  std::unordered_map<std::string, PackedW> packed;
  std::unordered_map<std::string, NormW> norms;
  std::unordered_map<std::string, XattnW> xattns;
  std::unordered_map<std::string, DirectW> directs;
  std::unordered_map<std::string, float*> v_biases;
  std::unordered_map<std::string, float*> f32s;
  std::vector<float> temb;   // [1280] time embedding for the configured timestep
  // Per-call fix_timesteps (genpercept_pipeline.py:405-408): the timestep only enters through
  // conv1.bias + time_emb_proj(silu(emb(t))) of the 22 UNet ResNets, so changing it re-folds those biases in place
  // (the device bias buffers keep their addresses: every plan and captured graph sees the new values).
  struct TembLayer { std::string key; std::vector<float> w, b, conv_bias; float* dev_bias = nullptr; int cout = 0; };
  std::vector<TembLayer> temb_layers;
  std::vector<float> te_w1, te_b1, te_w2, te_b2;
  std::map<int, std::vector<std::vector<float>>> temb_cache;   // timestep -> folded bias per layer
};

// engine.cu: pieces of the SD-2.1 UNet emitted on `b` over the weights `ws` holds under a checkpoint prefix.  The engine's
// graph and the per-kernel entry points (kernel_entry.cu) emit the same ops through them.
// ResnetBlock2D over concat(xs) (one or two sources) with 32 groups; temb_on folds the time embedding into conv1's bias.
// Returns a new arena tensor of `cout` channels whose GroupNorm statistics come with it where the epilogue makes them.
T4 resnet_block(Builder& b, WeightStore& ws, const std::string& p, const std::vector<T4>& xs, int cout, float eps, bool temb_on);
// out = x + attn2(norm2(x), context) of transformer block `blk`: the 2-token closed form when ws.n_tokens == 2, else LN ->
// scores GEMM -> per-head softmax -> output GEMM with the residual.
void cross_attention(Builder& b, WeightStore& ws, const std::string& blk, const T4& x, int heads, float eps, const T4& out);
// out [.., 4C] = GEGLU(ff.net.0.proj(x)) of transformer block `blk` (x [.., C], the projection's GEGLU epilogue)
void geglu_projection(Builder& b, WeightStore& ws, const std::string& blk, const T4& x, const T4& out);

// SD-2.1's CLIP text tower (transformers' CLIPTextModel, SURVEY.md App. A): token + position embedding, 23 pre-LN layers
// of causal self-attention (16 heads of 64) and an exact-erf GELU MLP, final LayerNorm.  Its weights are `text.` + the
// CLIPTextModel state-dict keys.
constexpr int kTextVocab = 49408, kTextDim = 1024, kTextLayers = 23, kTextHeads = 16, kTextMlp = 4096;
// The key -> shape of every tensor the tower reads.
const std::map<std::string, std::vector<int64_t>>& text_tower_spec();
// last_hidden_state [n, kTextDim] (fp32, `out`) of the n <= kTextMaxTokens token ids at `ids` (device), on the arena of `b`
void text_tower(Builder& b, WeightStore& ws, int n, const int32_t* ids, float* out);

// arena.cu: the per-device activation arena shared by the plans of engines with gp_set_shared_arena on.  join / leave
// count the engines that share it (the last leave unmaps everything and frees the reservation); add maps enough for a
// plan of `bytes` and returns the pool's fixed base, or null when the device cannot back it; remove gives a plan's share
// back, synchronising the device before it unmaps.  wait / record order a call's stream after every earlier user of the
// pool and every later user after the call.  record runs as a call's use of the arena ends, on a throw too, so it never
// throws: a failed record is left to the call's own CUDA error.
void shared_arena_join(int device);
void shared_arena_leave(int device);
uint8_t* shared_arena_add(int device, size_t bytes);
void shared_arena_remove(int device, size_t bytes);
void shared_arena_wait(int device, cudaStream_t s);
void shared_arena_record(int device, cudaStream_t s) noexcept;

// builder.cu: (BN, MT) of a stride-1 implicit-GEMM layer (default policy + the waves / L2-traffic model)
// N tile width for a GEMM with `cout` output columns (`force` != 0: that width); one of 16, 32, 64, 128.
int choose_bn(int cout, int force);
void tile_shape_for(int cout, double k_elems, bool tokens_mode, int images, int gw, int gh, int num_sms, int* bn, int* mt);
bool patch_tile_fits(int images, int h, int w, int cin, int csc, int cout, int bn, int mt, int num_sms);

}  // namespace gp
