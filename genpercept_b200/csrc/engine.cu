// The engine: the SD-2.1 GenPercept graph (VAE encoder -> UNet(t, empty-text) -> VAE decoder | DPT head) expressed
// on the Builder over the weights of a WeightStore (weights.cu), plan cache, CUDA-graph execution and the C-ABI.
//
// Graph semantics follow the reference call sites:
//   /root/reference/genpercept/genpercept_pipeline.py:375-526 (single_infer / encode_rgb / decode_pred)
//   /root/reference/genpercept/models/custom_unet.py:146-170,273,305-327,341-352,369-415
//   /root/reference/genpercept/models/dpt_head.py:52-90,213-335,338-388,530-546,564-592
// and the diffusers block definitions restated in SURVEY.md Appendix A.
#include <cstdlib>
#include <cstring>
#include <memory>
#include <tuple>

#include "engine.h"

using namespace gp;

namespace {

const int kUnetOut[4] = {320, 640, 1280, 1280};
const int kUnetHeads[4] = {5, 10, 20, 20};

bool is_set(const T4& t) { return t.off >= 0; }

}  // namespace

namespace gp {

T4 resnet_block(Builder& b, WeightStore& ws, const std::string& p, const std::vector<T4>& xs, int cout, float eps, bool temb_on) {
  int cin = 0;
  std::vector<int> cs;
  for (auto& x : xs) { cin += x.C; cs.push_back(x.C); }
  const T4& x0 = xs[0];
  // norm1 -> SiLU -> conv1 and norm2 -> SiLU -> conv2: the normalisation is an attribute of the convolution, which
  // Builder::conv materialises before it convolves
  T4 h = b.alloc(x0.N, x0.H, x0.W, cout);
  {
    ConvArgs c;
    c.srcs = xs;
    c.gn = &ws.norm_w(p + ".norm1"); c.gn_name = p + ".norm1"; c.gn_eps = eps;
    c.w = &ws.resnet_conv1(p, cin, temb_on);
    c.out = h;
    c.want_stats = true;     // feeds norm2
    b.conv(p + ".conv1", c);
  }
  T4 out = b.alloc(x0.N, x0.H, x0.W, cout);
  {
    ConvArgs c;
    c.srcs = {h};
    c.gn = &ws.norm_w(p + ".norm2"); c.gn_name = p + ".norm2"; c.gn_eps = eps;
    c.out = out;
    c.want_stats = true;     // resnet outputs feed the next GroupNorm (norm1 / transformer norm / conv_norm_out)
    if (cin != cout) {
      c.sc = xs;
      c.w = &ws.conv_w(p + ".conv2", {cout}, p + ".conv_shortcut", cs);
    } else {
      c.w = &ws.conv_w(p + ".conv2", {cout});
      c.res1 = &xs[0];
    }
    b.conv(p + ".conv2", c);
  }
  b.release(h);
  return out;
}

void cross_attention(Builder& b, WeightStore& ws, const std::string& blk, const T4& x, int heads, float eps, const T4& out) {
  if (ws.n_tokens == 2) {   // 2-token closed form, fused with its LayerNorm and residual
    b.xattn(blk + ".attn2", x, ws.xattn_w(blk, x.C, heads), eps, out);
    return;
  }
  // general context length: LN -> [C -> heads*n] GEMM -> per-head softmax -> [heads*n -> C] GEMM + residual
  const WeightStore::XattnGen xg = ws.xattn_general_w(blk, x.C, heads);
  T4 l2 = b.alloc(x.N, x.H, x.W, x.C);
  b.ln(blk + ".norm2", x, ws.norm_w(blk + ".norm2"), eps, l2);
  T4 sc = b.alloc(x.N, x.H, x.W, xg.Kp);
  { ConvArgs c; c.srcs = {l2}; c.ks = 1; c.w = xg.A; c.out = sc; b.conv(blk + ".attn2.scores", c); }
  b.release(l2);
  if (!b.measuring()) {
    void* sp = b.ptr(sc);
    const long long rows = x.pixels();
    const int kp = xg.Kp, nh = heads, nt = ws.n_tokens;
    const bool bf = b.bf16(), spl = b.split();
    b.custom(blk + ".attn2.softmax", 1, 2.0 * rows * kp * 2,
             [=](cudaStream_t s) { return softmax_groups(sp, rows, kp, nh, nt, bf, s, spl); });
  }
  { ConvArgs c; c.srcs = {sc}; c.ks = 1; c.w = xg.B; c.out = out; c.res1 = &x; b.conv(blk + ".attn2.out", c); }
  b.release(sc);
}

void geglu_projection(Builder& b, WeightStore& ws, const std::string& blk, const T4& x, const T4& out) {
  ConvArgs c; c.srcs = {x}; c.ks = 1; c.w = &ws.geglu_w(blk, x.C); c.out = out; c.cout_valid = 8 * x.C;
  c.flags = IG_GEGLU; c.force_bn = 128;
  b.conv(blk + ".ff.proj_geglu", c);
}

// transformers' CLIPTextTransformer.forward with causal masking and no padding mask (the reference tokenizes with
// padding='do_not_pad'): genpercept_pipeline.py:360-372
void text_tower(Builder& b, WeightStore& ws, int n, const int32_t* ids, float* out) {
  GP_REQUIRE(n >= 1 && n <= kTextMaxTokens, "text tower: 1 to " + std::to_string(kTextMaxTokens) + " tokens");
  const int D = kTextDim;
  const std::string m = "text.text_model.";
  const bool bf = b.bf16(), sp = b.split();
  const float* tok = ws.f32_w(m + "embeddings.token_embedding.weight");
  const float* pos = ws.f32_w(m + "embeddings.position_embedding.weight");
  T4 x = b.alloc(1, 1, n, D);
  if (!b.measuring()) {
    void* xp = b.ptr(x);
    b.custom(m + "embeddings", 1, (double)n * D * 8 + (double)x.bytes(),
             [=](cudaStream_t s) { return text_embed(ids, n, tok, pos, xp, D, bf, s, sp); });
  }
  for (int i = 0; i < kTextLayers; ++i) {
    const std::string p = m + "encoder.layers." + std::to_string(i);
    T4 l = b.alloc(1, 1, n, D);
    b.ln(p + ".layer_norm1", x, ws.norm_w(p + ".layer_norm1"), 1e-5f, l);
    T4 qkv = b.alloc(1, 1, n, 3 * D);
    { ConvArgs c; c.srcs = {l}; c.ks = 1; c.w = &ws.text_qkv_w(p + ".self_attn"); c.out = qkv; b.conv(p + ".self_attn.qkv", c); }
    b.release(l);
    T4 a = b.alloc(1, 1, n, D);
    if (!b.measuring()) {
      const void* qp = b.ptr(qkv);
      void* ap = b.ptr(a);
      b.custom(p + ".self_attn.causal", 1, (double)qkv.bytes() + (double)a.bytes(),
               [=](cudaStream_t s) { return causal_attention(qp, n, kTextHeads, D / kTextHeads, ap, bf, s, sp); });
    }
    b.release(qkv);
    T4 x1 = b.alloc(1, 1, n, D);
    { ConvArgs c; c.srcs = {a}; c.ks = 1; c.w = &ws.lin_w(p + ".self_attn.out_proj"); c.out = x1; c.res1 = &x; b.conv(p + ".self_attn.out_proj", c); }
    b.release(a);
    b.release(x);
    l = b.alloc(1, 1, n, D);
    b.ln(p + ".layer_norm2", x1, ws.norm_w(p + ".layer_norm2"), 1e-5f, l);
    T4 h = b.alloc(1, 1, n, kTextMlp);
    { ConvArgs c; c.srcs = {l}; c.ks = 1; c.w = &ws.lin_w(p + ".mlp.fc1"); c.out = h; b.conv(p + ".mlp.fc1", c); }
    b.release(l);
    T4 g = b.alloc(1, 1, n, kTextMlp);
    if (!b.measuring()) {
      const void* hp = b.ptr(h);
      void* gq = b.ptr(g);
      b.custom(p + ".mlp.gelu", 1, 2.0 * h.bytes(),
               [=](cudaStream_t s) { return gelu16(hp, gq, (long long)n * kTextMlp, bf, s, sp ? kTextMlp : 0); });
    }
    b.release(h);
    x = b.alloc(1, 1, n, D);
    { ConvArgs c; c.srcs = {g}; c.ks = 1; c.w = &ws.lin_w(p + ".mlp.fc2"); c.out = x; c.res1 = &x1; b.conv(p + ".mlp.fc2", c); }
    b.release(g);
    b.release(x1);
  }
  const NormW& fn = ws.norm_w(m + "final_layer_norm");
  if (!b.measuring()) {
    const void* xp = b.ptr(x);
    b.custom(m + "final_layer_norm", 1, (double)x.bytes() + (double)n * D * 4,
             [=](cudaStream_t s) { return layernorm_f32(xp, out, n, D, fn.gamma, fn.beta, 1e-5f, bf, s, sp); });
  }
  b.release(x);
}

}  // namespace gp

namespace {

struct Plan {
  int B = 0, H = 0, W = 0;
  uint8_t* arena = nullptr;
  size_t arena_bytes = 0;
  bool shared = false;              // the arena is the device's shared pool (gp_set_shared_arena), not the plan's own
  int device = 0;
  std::vector<Op> ops;
  // Arena tensors the entry points address.  A plan lacks (!is_set) z with the DPT readout, feat with the VAE readout
  // and xin .. x0 on the one-step arch.
  T4 rgb, rgb_latent, z, xin, sample, noise_pred, x0, feat[4];
  void* in_staging = nullptr;       // raw user input copy [B,3,H,W] (<= 4 bytes/elt), host inputs only
  float* out_f32 = nullptr;         // [B,3,outH,outW]: the plan's own result buffer (graph replay, host outputs, stage runs)
  float* out_dst = nullptr;         // where the final kernels write THIS launch (the caller's device buffer or out_f32);
                                    // read by the ops at launch time through Builder::out_slot
  int outH = 0, outW = 0;           // result extent: 8 * floor(H/8) (VAE readout), 64 * ceil-pyramid (DPT readout)
  uint64_t last_used = 0;
  // by (first stage, out_channels): gp_infer's and gp_infer_latent's ranges each have their own graphs and, per first
  // stage, their own first pass, which runs eagerly (kernel attributes, lazy init)
  std::map<std::pair<int, int>, cudaGraphExec_t> graphs;
  std::map<int, int> eager_runs;
  // gp_infer_steps' whole denoising loops, by (n_steps, noise given, out_channels); each key's first pass runs eagerly
  std::map<std::tuple<int, int, int>, cudaGraphExec_t> step_graphs;
  std::map<std::tuple<int, int, int>, int> step_eager_runs;
  double igemm_flops = 0;
  int64_t launches = 0;

  Plan() = default;
  Plan(const Plan&) = delete;
  Plan& operator=(const Plan&) = delete;
  void drop_step_graphs() {
    for (auto& g : step_graphs) cudaGraphExecDestroy(g.second);
    step_graphs.clear();
  }
  ~Plan() {
    drop_step_graphs();
    for (auto& g : graphs) cudaGraphExecDestroy(g.second);
    if (shared) shared_arena_remove(device, arena_bytes);
    else if (arena) cudaFree(arena);
  }
};

// Orders one entry point's use of a shared plan's arena after every earlier user of the pool, whatever its engine or
// stream, and before every later one: one event wait when the call starts, one record when it ends (on a throw too).
struct ArenaUse {
  const Plan* p;
  cudaStream_t s;
  ArenaUse(const Plan* plan, cudaStream_t st) : p(plan), s(st) { if (p->shared) shared_arena_wait(p->device, s); }
  ~ArenaUse() { if (p->shared) shared_arena_record(p->device, s); }
};

// The UNet's 22 time-embedded ResNets (the conv1 biases a timestep changes) in the order of a step's bias row: down
// blocks, mid block, up blocks, as unet() emits them.  (name, Cout).
std::vector<std::pair<std::string, int>> step_bias_layout() {
  std::vector<std::pair<std::string, int>> l;
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 2; ++j)
      l.emplace_back("unet.down_blocks." + std::to_string(i) + ".resnets." + std::to_string(j), kUnetOut[i]);
  for (int j = 0; j < 2; ++j) l.emplace_back("unet.mid_block.resnets." + std::to_string(j), 1280);
  const int up_out[4] = {1280, 1280, 640, 320};
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 3; ++j)
      l.emplace_back("unet.up_blocks." + std::to_string(i) + ".resnets." + std::to_string(j), up_out[i]);
  return l;
}

// gp_infer_steps' per-step data on the device, one set per engine.  Row i of `table` holds step i's folded conv1 biases
// in step_bias_layout order (`nbias` floats), then its four DDIM coefficients.  A call folds its rows on the host into
// the pinned `staging` buffer and uploads them on its stream; before each step's UNet ops, bias_scatter copies that
// step's row into the live bias buffers (`segs`).  So a captured loop reads the call's timesteps and coefficients as
// data: nothing in it depends on them.
struct StepTables {
  std::vector<std::string> keys;     // the ResNet of each segment
  std::vector<BiasSegment> host_segs;
  BiasSegment* segs = nullptr;       // device copy of host_segs
  int nbias = 0, row = 0;            // floats of biases per step, floats per row (nbias + 4)
  int cap = 0;                       // rows of `table` and `staging`
  float* table = nullptr;            // device [cap][row]
  float* staging = nullptr;          // pinned host [cap][row]
  cudaEvent_t staged = nullptr;      // recorded after the last upload from `staging`
  cudaEvent_t released = nullptr;    // recorded after the last call's work: its reads of `table` and the bias buffers,
                                     // and the hand-off of its result from out_f32

  StepTables() = default;
  StepTables(const StepTables&) = delete;
  StepTables& operator=(const StepTables&) = delete;
  ~StepTables() {
    if (released) cudaEventSynchronize(released);
    if (staged) cudaEventSynchronize(staged);
    if (table) cudaFree(table);
    if (staging) cudaFreeHost(staging);
    if (segs) cudaFree(segs);
    if (staged) cudaEventDestroy(staged);
    if (released) cudaEventDestroy(released);
  }

  // Binds the layout to the store's bias buffers (after gp_finalize packed every weight): each of the 22 buffers once.
  void init(const WeightStore& ws) {
    int off = 0;
    for (const auto& [key, cout] : step_bias_layout()) {
      int rows = 0;
      float* slot = ws.temb_bias_slot(key, &rows);
      GP_REQUIRE(slot && rows == cout, key + ": no time-embedded conv1 bias of " + std::to_string(cout) + " channels");
      keys.push_back(key);
      host_segs.push_back(BiasSegment{slot, off, cout});
      off += cout;
    }
    GP_REQUIRE(ws.temb_slot_count() == (int)host_segs.size(), "the UNet has time-embedded ResNets outside the step layout");
    nbias = off;
    row = nbias + 4;
    const size_t bytes = host_segs.size() * sizeof(BiasSegment);
    GP_CUDA(cudaMalloc(reinterpret_cast<void**>(&segs), bytes));
    GP_CUDA(cudaMemcpy(segs, host_segs.data(), bytes, cudaMemcpyHostToDevice));
    GP_CUDA(cudaEventCreateWithFlags(&staged, cudaEventDisableTiming));
    GP_CUDA(cudaEventCreateWithFlags(&released, cudaEventDisableTiming));
  }
};

// gp_encode_text's tower for one token count: its own arena (the ids, the fp32 result, then the activations) and ops.
struct TextPlan {
  uint8_t* arena = nullptr;
  int32_t* ids = nullptr;
  float* out = nullptr;
  std::vector<Op> ops;
  TextPlan() = default;
  TextPlan(const TextPlan&) = delete;
  TextPlan& operator=(const TextPlan&) = delete;
  ~TextPlan() { if (arena) cudaFree(arena); }
};

// The text tower of an engine until gp_finalize: the text.* checkpoint tensors, the device weights packed from them (a
// store of its own, outside the image plans' weight bytes) and a plan per token count.
struct TextTower {
  std::unique_ptr<WeightStore> ws;
  std::map<int, std::unique_ptr<TextPlan>> plans;
  bool packed = false;        // ws holds device weights

  // The plan for n tokens: the measuring pass sizes the arena (and packs the weights on first use), the second emits.
  TextPlan* plan(int n) {
    auto it = plans.find(n);
    if (it != plans.end()) return it->second.get();
    auto emit = [&](Builder& b, TextPlan* p) {
      const size_t ids_off = b.raw_alloc((size_t)kTextMaxTokens * sizeof(int32_t));
      const size_t out_off = b.raw_alloc((size_t)n * kTextDim * sizeof(float));
      if (p) {
        p->ids = reinterpret_cast<int32_t*>(b.raw_ptr(ids_off));
        p->out = reinterpret_cast<float*>(b.raw_ptr(out_off));
      }
      text_tower(b, *ws, n, p ? p->ids : nullptr, p ? p->out : nullptr);
    };
    Builder m(ws->bf16, true, nullptr, ws->split);
    packed = true;
    emit(m, nullptr);
    std::unique_ptr<TextPlan> p(new TextPlan());
    GP_CUDA(cudaMalloc(reinterpret_cast<void**>(&p->arena), m.arena_bytes()));
    Builder b(ws->bf16, false, p->arena, ws->split);
    emit(b, p.get());
    if (b.arena_bytes() != m.arena_bytes()) throw GpError(GP_ERR_STATE, "text tower: planner passes disagree on arena size");
    p->ops = std::move(b.ops);
    return plans.emplace(n, std::move(p)).first->second.get();
  }
};

}  // namespace

struct gp_engine {
  gp_config cfg;
  std::string err;
  bool poisoned = false, finalized = false;
  WeightStore ws;
  bool multistep = false;    // cfg.arch == 1: real DDIM steps around the UNet (SURVEY.md §8 f4), no scheduler fold
  int unet_in_ch = 0;        // 4, or 8 for the marigold arch (cat([rgb_latent, pred_latent]))
  uint64_t use_clock = 0;
  std::map<std::tuple<int, int, int>, std::unique_ptr<Plan>> plans;
  Plan* cur = nullptr;
  bool mem_efficient_attn = false;   // gp_set_memory_efficient_attention: fused attention in the high-precision mode
  bool shared_arena = false;         // gp_set_shared_arena: new plans take their arena from the device's shared pool
  StepTables steps;                  // the multi-step arch's per-step biases and coefficients (gp_infer_steps)
  TextTower text;                    // gp_encode_text until gp_finalize

  ~gp_engine() {
    if (!shared_arena) return;
    cudaSetDevice(cfg.device);
    plans.clear();             // each shared plan gives its share back before the engine leaves the pool
    shared_arena_leave(cfg.device);
  }

  // Synchronises, then drops a cached plan (its graph execs and arena go with it).
  void drop_plan(std::map<std::tuple<int, int, int>, std::unique_ptr<Plan>>::iterator it) {
    GP_CUDA(cudaDeviceSynchronize());
    if (cur == it->second.get()) cur = nullptr;
    plans.erase(it);
  }

  // Makes room for `n` rows in the step tables.  Growing frees the old table, so the graphs that read it go too; the host
  // waits only for the last call that used it.
  void reserve_steps(int n) {
    StepTables& st = steps;
    if (n <= st.cap) return;
    const int cap = std::max(n, 2 * st.cap);
    GP_CUDA(cudaEventSynchronize(st.released));
    GP_CUDA(cudaEventSynchronize(st.staged));
    for (auto& kv : plans) kv.second->drop_step_graphs();
    if (st.table) GP_CUDA(cudaFree(st.table));
    if (st.staging) GP_CUDA(cudaFreeHost(st.staging));
    st.table = nullptr;
    st.staging = nullptr;
    st.cap = 0;
    const size_t bytes = (size_t)cap * st.row * sizeof(float);
    GP_CUDA(cudaMalloc(reinterpret_cast<void**>(&st.table), bytes));
    GP_CUDA(cudaMallocHost(reinterpret_cast<void**>(&st.staging), bytes));
    st.cap = cap;
  }

  // ------------------------------------------------------------------ graph pieces
  // 3x3 conv whose input is an NHWC8 tensor with `cin` (4 or 8) real channels: one 64-wide K chunk
  // per tap through the tensor-core kernel (the TMA box zero-fills channels >= 8).
  void small_cin_conv(Builder& b, const std::string& key, const T4& src8, int cin, const T4& out) {
    ConvArgs c;
    c.srcs = {src8};
    c.w = &ws.conv_w(key, {cin});
    c.out = out;
    c.want_stats = true;
    b.conv(key, c);
  }

  T4 transformer(Builder& b, const std::string& p, const T4& x, int heads) {
    const int C = x.C;
    const std::string blk = p + ".transformer_blocks.0";
    T4 n = b.alloc(x.N, x.H, x.W, C);
    b.gn(p + ".norm", {x}, ws.norm_w(p + ".norm"), 32, 1e-6f, false, n);
    T4 t = b.alloc(x.N, x.H, x.W, C);
    { ConvArgs c; c.srcs = {n}; c.ks = 1; c.w = &ws.lin_w(p + ".proj_in"); c.out = t; b.conv(p + ".proj_in", c); }
    b.release(n);
    // self attention
    T4 l = b.alloc(x.N, x.H, x.W, C);
    b.ln(blk + ".norm1", t, ws.norm_w(blk + ".norm1"), 1e-5f, l);
    T4 o = b.alloc(x.N, x.H, x.W, C);
    b.attention(blk + ".attn1", l, ws.self_attn_qk(blk, C, heads), ws.lin_w(blk + ".attn1.to_v", false), nullptr, heads, o);
    b.release(l);
    T4 t1 = b.alloc(x.N, x.H, x.W, C);
    { ConvArgs c; c.srcs = {o}; c.ks = 1; c.w = &ws.lin_w(blk + ".attn1.to_out.0"); c.out = t1; c.res1 = &t; b.conv(blk + ".attn1.to_out", c); }
    b.release(o);
    b.release(t);
    // cross attention
    T4 t2 = b.alloc(x.N, x.H, x.W, C);
    cross_attention(b, ws, blk, t1, heads, 1e-5f, t2);
    b.release(t1);
    // feed-forward (GEGLU)
    T4 l3 = b.alloc(x.N, x.H, x.W, C);
    b.ln(blk + ".norm3", t2, ws.norm_w(blk + ".norm3"), 1e-5f, l3);
    T4 gg = b.alloc(x.N, x.H, x.W, 4 * C);
    geglu_projection(b, ws, blk, l3, gg);
    b.release(l3);
    T4 t3 = b.alloc(x.N, x.H, x.W, C);
    { ConvArgs c; c.srcs = {gg}; c.ks = 1; c.w = &ws.lin_w(blk + ".ff.net.2"); c.out = t3; c.res1 = &t2; b.conv(blk + ".ff.out", c); }
    b.release(gg);
    b.release(t2);
    T4 out = b.alloc(x.N, x.H, x.W, C);
    { ConvArgs c; c.srcs = {t3}; c.ks = 1; c.w = &ws.lin_w(p + ".proj_out"); c.out = out; c.res1 = &x; c.want_stats = true; b.conv(p + ".proj_out", c); }
    b.release(t3);
    return out;
  }

  T4 vae_mid(Builder& b, const std::string& p, T4 x) {
    T4 r0 = resnet_block(b, ws,p + ".resnets.0", {x}, 512, 1e-6f, false);
    b.release(x);
    const std::string a = p + ".attentions.0";
    T4 n = b.alloc(r0.N, r0.H, r0.W, 512);
    b.gn(a + ".group_norm", {r0}, ws.norm_w(a + ".group_norm"), 32, 1e-6f, false, n);
    T4 o = b.alloc(r0.N, r0.H, r0.W, 512);
    b.attention(a, n, ws.vae_attn_qk(a), ws.lin_w(a + ".to_v", false), ws.vae_v_bias(a), 1, o);
    b.release(n);
    T4 y = b.alloc(r0.N, r0.H, r0.W, 512);
    { ConvArgs c; c.srcs = {o}; c.ks = 1; c.w = &ws.lin_w(a + ".to_out.0"); c.out = y; c.res1 = &r0; c.want_stats = true; b.conv(a + ".to_out", c); }
    b.release(o);
    b.release(r0);
    T4 r1 = resnet_block(b, ws,p + ".resnets.1", {y}, 512, 1e-6f, false);
    b.release(y);
    return r1;
  }

  // encode_rgb: genpercept_pipeline.py:488-505
  T4 vae_encoder(Builder& b, const T4& rgb32) {
    const std::string e = "vae.encoder";
    T4 x = b.alloc(rgb32.N, rgb32.H, rgb32.W, 128);
    {   // conv_in over the K-packed input (preprocess_rgb_im2col): a 1x1 GEMM with K = 27
      ConvArgs c;
      c.srcs = {rgb32};
      c.ks = 1;
      c.w = &ws.encoder_conv_in();
      c.out = x;
      c.want_stats = true;
      b.conv(e + ".conv_in", c);
    }
    const int ch[5] = {128, 128, 256, 512, 512};
    for (int i = 0; i < 4; ++i) {
      for (int j = 0; j < 2; ++j) {
        T4 y = resnet_block(b, ws,e + ".down_blocks." + std::to_string(i) + ".resnets." + std::to_string(j), {x}, ch[i + 1], 1e-6f, false);
        b.release(x);
        x = y;
      }
      if (i < 3) {
        const std::string k = e + ".down_blocks." + std::to_string(i) + ".downsamplers.0.conv";
        const auto [Ho, Wo] = conv_out_dims(2, x.H, x.W);
        T4 y = b.alloc(x.N, Ho, Wo, x.C);
        ConvArgs c; c.srcs = {x}; c.mode = 2; c.w = &ws.conv_w(k, {x.C}); c.out = y; c.want_stats = true;
        b.conv(k, c);
        b.release(x);
        x = y;
      }
    }
    x = vae_mid(b, e + ".mid_block", x);
    // conv_out o quant_conv, mean channels, * 0.18215: one 3x3 conv 512->4 (WeightStore::encoder_tail)
    T4 lat = b.alloc(x.N, x.H, x.W, 8);
    {
      ConvArgs c; c.srcs = {x}; c.w = &ws.encoder_tail(); c.out = lat;
      c.gn = &ws.norm_w(e + ".conv_norm_out"); c.gn_name = e + ".conv_norm_out"; c.gn_eps = 1e-6f;
      b.conv("vae.encoder.tail", c);
    }
    b.release(x);
    return lat;
  }

  // UNet2DConditionModel.forward (custom_unet.py); returns z (NHWC8) or, for the DPT readout, the 4 taps
  void unet(Builder& b, const T4& lat8, bool want_feats, T4* z_out, T4 feats[4]) {
    ws.compute_temb(cfg.timestep);
    const std::string u = "unet";
    T4 x = b.alloc(lat8.N, lat8.H, lat8.W, 320);
    if (unet_in_ch == 0) {
      unet_in_ch = ws.unet_in_channels();
      GP_REQUIRE(multistep || unet_in_ch == 4, "an 8-channel conv_in belongs to the multi-step arch (gp_config.arch = 1)");
    }
    small_cin_conv(b, u + ".conv_in", lat8, unet_in_ch, x);
    std::vector<T4> skips = {x};
    for (int i = 0; i < 4; ++i) {
      const int cout = kUnetOut[i];
      for (int j = 0; j < 2; ++j) {
        const std::string rp = u + ".down_blocks." + std::to_string(i) + ".resnets." + std::to_string(j);
        T4 y = resnet_block(b, ws,rp, {x}, cout, 1e-5f, true);
        if (i < 3) {
          T4 y2 = transformer(b, u + ".down_blocks." + std::to_string(i) + ".attentions." + std::to_string(j), y, kUnetHeads[i]);
          b.release(y);
          y = y2;
        }
        x = y;
        skips.push_back(x);
      }
      if (i < 3) {
        const std::string k = u + ".down_blocks." + std::to_string(i) + ".downsamplers.0.conv";
        const auto [Ho, Wo] = conv_out_dims(1, x.H, x.W);
        T4 y = b.alloc(x.N, Ho, Wo, x.C);
        ConvArgs c; c.srcs = {x}; c.mode = 1; c.w = &ws.conv_w(k, {x.C}); c.out = y; c.want_stats = true;
        b.conv(k, c);
        x = y;
        skips.push_back(x);
      }
    }
    // mid block; x (the last skip) stays alive for the up path
    T4 m0 = resnet_block(b, ws,u + ".mid_block.resnets.0", {x}, 1280, 1e-5f, true);
    T4 m1 = transformer(b, u + ".mid_block.attentions.0", m0, 20);
    b.release(m0);
    T4 cur = resnet_block(b, ws,u + ".mid_block.resnets.1", {m1}, 1280, 1e-5f, true);
    b.release(m1);
    const int up_out[4] = {1280, 1280, 640, 320};
    const bool up_attn[4] = {false, true, true, true};
    const int up_heads[4] = {0, 20, 10, 5};
    for (int i = 0; i < 4; ++i) {
      for (int j = 0; j < 3; ++j) {
        T4 skip = skips.back();
        skips.pop_back();
        const std::string rp = u + ".up_blocks." + std::to_string(i) + ".resnets." + std::to_string(j);
        T4 y = resnet_block(b, ws,rp, {cur, skip}, up_out[i], 1e-5f, true);
        b.release(cur);
        b.release(skip);
        if (up_attn[i]) {
          T4 y2 = transformer(b, u + ".up_blocks." + std::to_string(i) + ".attentions." + std::to_string(j), y, up_heads[i]);
          b.release(y);
          y = y2;
        }
        cur = y;
      }
      if (i < 3) {
        // Upsample2D: nearest resize to the skip's size + 3x3 conv.  Exact 2x (every level, when H and W are
        // multiples of 64): the fused four-class 2x2 form.  Otherwise (a level with an odd extent: the target is
        // 2n-1, diffusers' `upsample_size`) the resized tensor is materialised and the plain 3x3 weights are used —
        // the pre-summed 2x2 weights would be wrong in the last row / column, where the padding cuts the window.
        const T4 nxt = skips.back();
        const std::string k = u + ".up_blocks." + std::to_string(i) + ".upsamplers.0.conv";
        const PackedW& plain = ws.conv_w(k, {cur.C}, "", {}, nullptr, true, "#plain");   // packed at finalize for both paths
        if (nxt.H == 2 * cur.H && nxt.W == 2 * cur.W) {
          T4 y = b.alloc(cur.N, 2 * cur.H, 2 * cur.W, cur.C);
          ConvArgs c; c.srcs = {cur}; c.mode = 3; c.w = &ws.conv_up_w(k); c.out = y; c.want_stats = true;
          b.conv(k, c);
          b.release(cur);
          cur = y;
        } else {
          GP_REQUIRE(nxt.H <= 2 * cur.H && nxt.H >= 2 * cur.H - 1 && nxt.W <= 2 * cur.W && nxt.W >= 2 * cur.W - 1,
                     "unexpected skip size in the UNet up path");
          T4 up = b.alloc(cur.N, nxt.H, nxt.W, cur.C);
          b.resize(k + ".nearest", cur, up, true);
          b.release(cur);
          T4 y = b.alloc(up.N, up.H, up.W, up.C);
          ConvArgs c; c.srcs = {up}; c.mode = 0; c.w = &plain; c.out = y; c.want_stats = true;
          b.conv(k, c);
          b.release(up);
          cur = y;
        }
      }
      if (want_feats) {
        // custom_unet.py:400 taps each up block's output (after its upsampler); keep them alive
        T4 f = b.alloc(cur.N, cur.H, cur.W, cur.C);
        feats[i] = f;
        if (!b.measuring()) {
          void* dst = b.ptr(f);
          const void* src = b.ptr(cur);
          const size_t nb = cur.bytes();
          b.custom(u + ".feat_tap" + std::to_string(i), 1, 2.0 * nb,
                   [=](cudaStream_t s) { return cudaMemcpyAsync(dst, src, nb, cudaMemcpyDeviceToDevice, s); });
        }
      }
    }
    if (want_feats) {
      b.release(cur);
      return;
    }
    if (multistep) {   // the scheduler step is a real one: conv_out as it is (model_output), DDIM + post_quant_conv run outside
      ConvArgs c; c.srcs = {cur}; c.w = &ws.unet_conv_out_plain(); c.out = *z_out;
      c.gn = &ws.norm_w(u + ".conv_norm_out"); c.gn_name = u + ".conv_norm_out"; c.gn_eps = 1e-5f;
      b.conv("unet.conv_out", c);
      b.release(cur);
      return;
    }
    // conv_out, DDIM(beta=1) x0 = -v, /0.18215, post_quant_conv: one 3x3 conv 320->4 (WeightStore::unet_tail)
    {
      ConvArgs c; c.srcs = {cur}; c.w = &ws.unet_tail(); c.out = *z_out;
      c.gn = &ws.norm_w(u + ".conv_norm_out"); c.gn_name = u + ".conv_norm_out"; c.gn_eps = 1e-5f;
      b.conv("unet.tail", c);
    }
    b.release(cur);
  }

  // decode_pred + clip + shift: genpercept_pipeline.py:507-526, :470-472
  void vae_decoder(Builder& b, const T4& z8, float* out_f32) {
    const std::string d = "vae.decoder";
    T4 x = b.alloc(z8.N, z8.H, z8.W, 512);
    small_cin_conv(b, d + ".conv_in", z8, 4, x);
    x = vae_mid(b, d + ".mid_block", x);
    const int oc[4] = {512, 512, 256, 128};
    for (int i = 0; i < 4; ++i) {
      for (int j = 0; j < 3; ++j) {
        T4 y = resnet_block(b, ws,d + ".up_blocks." + std::to_string(i) + ".resnets." + std::to_string(j), {x}, oc[i], 1e-6f, false);
        b.release(x);
        x = y;
      }
      if (i < 3) {
        const std::string k = d + ".up_blocks." + std::to_string(i) + ".upsamplers.0.conv";
        T4 y = b.alloc(x.N, 2 * x.H, 2 * x.W, x.C);
        ConvArgs c; c.srcs = {x}; c.mode = 3; c.w = &ws.conv_up_w(k); c.out = y; c.want_stats = true;
        b.conv(k, c);
        b.release(x);
        x = y;
      }
    }
    // 3-channel (normal / seg) and channel-mean (depth / matting / dis / disparity) variants
    for (int variant : {1, 3}) {
      b.variant = variant;
      ConvArgs c;
      c.srcs = {x};
      c.gn = &ws.norm_w(d + ".conv_norm_out"); c.gn_name = d + ".conv_norm_out"; c.gn_eps = 1e-6f;
      c.w = variant == 1 ? &ws.decoder_tail1() : &ws.conv_w(d + ".conv_out", {128});
      c.out_f32 = out_f32;
      c.cout_valid = variant;
      c.flags = IG_AFFINE_CLAMP01;
      T4 shape = x;   // only N/H/W are consulted for fp32 outputs
      c.out = shape;
      b.conv("vae.decoder.tail" + std::to_string(variant), c);
    }
    b.variant = 0;
    b.release(x);
  }

  // DPTNeckHeadForUnetAfterUpsampleIdentity (dpt_head.py:530-546), then per-image min-max (:482, F12)
  T4 dpt_rcu(Builder& b, const std::string& p, const T4& x, const T4* extra_res) {
    T4 r = b.alloc(x.N, x.H, x.W, 256);
    b.relu_op(p + ".relu", x, r);
    T4 c1 = b.alloc(x.N, x.H, x.W, 256);
    { ConvArgs c; c.srcs = {r}; c.w = &ws.conv_w(p + ".convolution1", {256}, "", {}, nullptr, false); c.out = c1; c.flags = IG_RELU; b.conv(p + ".convolution1", c); }
    b.release(r);
    T4 out = b.alloc(x.N, x.H, x.W, 256);
    { ConvArgs c; c.srcs = {c1}; c.w = &ws.conv_w(p + ".convolution2", {256}, "", {}, nullptr, false); c.out = out; c.res1 = &x; c.res2 = extra_res; b.conv(p + ".convolution2", c); }
    b.release(c1);
    return out;
  }
  void dpt_head(Builder& b, T4 feats[4], float* out_f32, unsigned int* mm_scratch, int* out_h, int* out_w) {
    // feats (up-block order): [1280@h/4, 1280@h/2, 640@h, 320@h]; reference reverses (:479)
    T4 f0 = feats[3], f1 = feats[2], f2 = feats[1], f3 = feats[0];
    T4 f0u = b.alloc(f0.N, 2 * f0.H, 2 * f0.W, 320);
    { ConvArgs c; c.srcs = {f0}; c.mode = 3; c.w = &ws.conv_up_w("dpt.feature_upsample_0.conv"); c.out = f0u; b.conv("dpt.feature_upsample_0", c); }
    const T4 fin[4] = {f0u, f1, f2, f3};
    T4 nk[4];
    for (int i = 0; i < 4; ++i) {
      nk[i] = b.alloc(fin[i].N, fin[i].H, fin[i].W, 256);
      ConvArgs c; c.srcs = {fin[i]}; c.w = &ws.conv_w("dpt.neck.convs." + std::to_string(i), {fin[i].C}, "", {}, nullptr, false); c.out = nk[i];
      b.conv("dpt.neck.convs." + std::to_string(i), c);
    }
    b.release(f0u);
    // fusion stage runs coarse -> fine: nk[3] (h/4), nk[2], nk[1], nk[0] (2h)
    T4 x{};
    for (int li = 0; li < 4; ++li) {
      const std::string lp = "dpt.neck.fusion_stage.layers." + std::to_string(li);
      const T4& f = nk[3 - li];
      T4 y;
      if (li == 0) {
        y = dpt_rcu(b, lp + ".residual_layer2", f, nullptr);
      } else {
        // dpt_head.py:297-300: a skip feature whose extent differs from the running map's (odd pyramid levels) is
        // resized to it, bilinear, align_corners=False
        T4 fr = f;
        const bool rs = x.H != f.H || x.W != f.W;
        if (rs) {
          fr = b.alloc(x.N, x.H, x.W, 256);
          b.resize(lp + ".resize_skip", f, fr, false);
        }
        T4 s = dpt_rcu(b, lp + ".residual_layer1", fr, &x);   // x + (f + conv2(...))
        if (rs) b.release(fr);
        b.release(x);
        y = dpt_rcu(b, lp + ".residual_layer2", s, nullptr);
        b.release(s);
      }
      b.release(f);
      T4 up = b.alloc(y.N, 2 * y.H, 2 * y.W, 256);
      b.bilinear(lp + ".up", y, up);
      b.release(y);
      x = b.alloc(up.N, up.H, up.W, 256);
      { ConvArgs c; c.srcs = {up}; c.ks = 1; c.w = &ws.lin_w(lp + ".projection"); c.out = x; b.conv(lp + ".projection", c); }
      b.release(up);
    }
    T4 p = b.alloc(x.N, x.H, x.W, 256);
    { ConvArgs c; c.srcs = {x}; c.w = &ws.conv_w("dpt.head.projection", {256}); c.out = p; c.flags = IG_RELU; b.conv("dpt.head.projection", c); }
    b.release(x);
    T4 h0 = b.alloc(p.N, p.H, p.W, 128);
    { ConvArgs c; c.srcs = {p}; c.w = &ws.conv_w("dpt.head.head.0", {256}); c.out = h0; b.conv("dpt.head.head.0", c); }
    b.release(p);
    T4 h1 = b.alloc(h0.N, 2 * h0.H, 2 * h0.W, 128);
    b.bilinear("dpt.head.up", h0, h1);
    b.release(h0);
    T4 h2 = b.alloc(h1.N, h1.H, h1.W, 32);
    { ConvArgs c; c.srcs = {h1}; c.w = &ws.conv_w("dpt.head.head.2", {128}); c.out = h2; c.flags = IG_RELU; b.conv("dpt.head.head.2", c); }
    b.release(h1);
    b.direct("dpt.head.head.4", h2, 32, ws.direct_w("dpt.head.head.4", 32), h2, out_f32);
    const int N = h2.N;
    const long long HW = (long long)h2.H * h2.W;
    *out_h = h2.H; *out_w = h2.W;
    b.release(h2);
    float** slot = b.out_slot;
    b.custom("dpt.minmax", 3, 3.0 * N * HW * 4, [=](cudaStream_t s) { return minmax_normalize(slot ? *slot : out_f32, N, HW, mm_scratch, s); });
  }

  void build(Builder& b, Plan* plan, int B, int H, int W) {
    // The VAE needs multiples of 8 (three stride-2 stages); the UNet handles odd latent extents like diffusers
    // (ceil on the way down, resize to the skip's size on the way up).  The DPT head's fusion stages assume
    // matching pyramid sizes: multiples of 64 there (the reference resizes the skip bilinearly otherwise).
    // Any H, W >= 32, like the reference: the VAE's stride-2 stages floor (asymmetric padding), so the decoded map is
    // 8*floor(H/8) x 8*floor(W/8); the DPT fusion stages resize a skip feature to the running map when the pyramid
    // extents differ (dpt_head.py:297-300), so its map is a multiple of 64 that covers the input.  __call__'s
    // match_input_res resize brings either back to the input size (genpercept_pipeline.py:301-307).
    // persistent buffers first so their offsets are identical in both passes
    const size_t in_off = b.raw_alloc((size_t)B * 3 * H * W * 4);
    const size_t out_off = b.raw_alloc((size_t)B * 3 * (H + 64) * (W + 64) * 4);
    const size_t ss_off = b.raw_alloc((size_t)B * 2560 * 2 * 4);
    const size_t mm_off = b.raw_alloc((size_t)B * 2 * 4);
    T4 rgb8 = b.alloc(B, H, W, 32);      // K-packed 3x3 neighbourhoods (preprocess_rgb_im2col); channels 0..2 = the image
    float* out_f32 = nullptr;
    if (!b.measuring()) {
      plan->in_staging = b.raw_ptr(in_off);
      plan->out_f32 = reinterpret_cast<float*>(b.raw_ptr(out_off));
      plan->out_dst = plan->out_f32;
      out_f32 = plan->out_f32;
      b.out_slot = &plan->out_dst;
      b.gn_ss = reinterpret_cast<float*>(b.raw_ptr(ss_off));
    }
    unsigned int* mm = b.measuring() ? nullptr : reinterpret_cast<unsigned int*>(b.raw_ptr(mm_off));
    b.stage = GP_STAGE_VAE_ENCODE;
    T4 latent = vae_encoder(b, rgb8);
    b.stage = GP_STAGE_UNET;
    const bool dpt = cfg.readout == GP_READOUT_DPT;
    T4 feats[4];
    T4 z = b.alloc(B, latent.H, latent.W, 8);
    T4 xin{}, sample{}, npred{}, x0{};
    if (multistep) {
      GP_REQUIRE(!dpt, "the multi-step archs decode with the VAE (the reference's DPT readout is one-step)");
      xin = b.alloc(B, latent.H, latent.W, 8);      // the UNet's input of a step
      sample = b.alloc(B, latent.H, latent.W, 8);   // pred_latent
      npred = b.alloc(B, latent.H, latent.W, 8);    // model_output
      x0 = b.alloc(B, latent.H, latent.W, 8);       // pred_original_sample
      unet(b, xin, false, &npred, feats);
    } else {
      unet(b, latent, dpt, &z, feats);
    }
    b.stage = GP_STAGE_READOUT;
    int oh = 8 * latent.H, ow = 8 * latent.W;
    if (dpt) dpt_head(b, feats, out_f32, mm, &oh, &ow);
    else vae_decoder(b, z, out_f32);
    GP_REQUIRE(oh <= H + 64 && ow <= W + 64, "result extent exceeds the plan's output buffer");
    if (!b.measuring()) {
      plan->outH = oh; plan->outW = ow;
      plan->rgb = rgb8;
      plan->rgb_latent = latent;
      if (!dpt) plan->z = z;
      if (multistep) {
        plan->xin = xin;
        plan->sample = sample;
        plan->noise_pred = npred;
        plan->x0 = x0;
      }
      if (dpt)
        for (int i = 0; i < 4; ++i) plan->feat[i] = feats[i];
    }
  }
};

// ------------------------------------------------------------------------------------ C-ABI
namespace {

template <class F>
gp_status guarded(gp_engine* e, F f) {
  if (!e) return GP_ERR_INVALID;
  if (e->poisoned) { e->err = "engine poisoned by an earlier CUDA error: " + e->err; return GP_ERR_CUDA; }
  const gp_status st = run_guarded(f, e->err);
  if (st == GP_ERR_CUDA) e->poisoned = true;
  return st;
}

cudaError_t run_ops(Plan* p, int stage_lo, int stage_hi, int out_channels, cudaStream_t s) {
  for (auto& op : p->ops) {
    if (op.stage < stage_lo || op.stage > stage_hi) continue;
    if (op.variant != 0 && op.variant != out_channels) continue;
    cudaError_t e = op.run(s);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

// The plan the run and inspection entry points work on; `fn` names the entry point in the error.
Plan* current_plan(gp_engine* e, const char* fn) {
  if (!e->cur) throw GpError(GP_ERR_NO_PLAN, std::string(fn) + ": no plan (call gp_plan)");
  return e->cur;
}

// Points the plan's final kernels at `dst` (the caller's device buffer or out_f32) for one run, and back at out_f32 when
// it leaves scope, on a throw too.
struct ResultTo {
  Plan* p;
  ResultTo(Plan* plan, float* dst) : p(plan) { p->out_dst = dst; }
  ~ResultTo() { p->out_dst = p->out_f32; }
  // Copies the result to the caller's `out` when the kernels wrote it to out_f32.
  void deliver(float* out, int out_on_host, int out_channels, cudaStream_t s) const {
    if (p->out_dst != out)
      GP_CUDA(cudaMemcpyAsync(out, p->out_f32, (size_t)p->B * p->outH * p->outW * out_channels * 4,
                              out_on_host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, s));
  }
};

// The caller's rgb (u8, f16 or f32) -> the plan's K-packed input.  A device input is read where it lies; only host inputs
// go through the plan's staging buffer.  `fn` names the entry point in the error message.
void stage_rgb(gp_engine* e, Plan* p, const void* rgb, int rgb_dtype, int rgb_on_host, cudaStream_t s, const char* fn) {
  int kind = 0;
  size_t esz = 1;
  if (rgb_dtype == GP_U8) { kind = 0; esz = 1; }
  else if (rgb_dtype == GP_F16) { kind = 1; esz = 2; }
  else if (rgb_dtype == GP_F32) { kind = 2; esz = 4; }
  else throw GpError(GP_ERR_INVALID, std::string(fn) + ": rgb dtype must be u8, f16 or f32");
  const void* src = rgb;
  if (rgb_on_host) {
    GP_CUDA(cudaMemcpyAsync(p->in_staging, rgb, (size_t)p->B * p->H * p->W * 3 * esz, cudaMemcpyHostToDevice, s));
    src = p->in_staging;
  }
  GP_CUDA(preprocess_rgb_im2col(src, kind, p->arena + p->rgb.off, p->B, p->H, p->W, e->ws.bf16, s, e->ws.split));
}

// Whether the plan's passes replay captured graphs: always (use_cuda_graph 1), or with 2 = auto where the launch stream is
// the bottleneck — small plans.
bool uses_graph(const gp_engine* e, const Plan* p) {
  return e->cfg.use_cuda_graph == 1 ||
         (e->cfg.use_cuda_graph == 2 && (long long)p->B * p->H * p->W <= 2LL * 768 * 768);
}

// Captures what `enqueue(stream)` launches into an executable graph.
template <class F>
cudaGraphExec_t capture_graph(F enqueue) {
  cudaStream_t cs;
  GP_CUDA(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
  cudaGraph_t g;
  GP_CUDA(cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal));
  cudaError_t re = enqueue(cs);
  cudaError_t ce = cudaStreamEndCapture(cs, &g);
  cudaStreamDestroy(cs);
  GP_CUDA(re);
  GP_CUDA(ce);
  cudaGraphExec_t ge;
  GP_CUDA(cudaGraphInstantiate(&ge, g, 0));
  cudaGraphDestroy(g);
  return ge;
}

// Runs the ops of stages `first` .. GP_STAGE_READOUT and delivers the result to `out` (device, or host if out_on_host).
// The first pass from `first` runs eagerly; with CUDA graphs on, later passes replay the graph captured for
// (first, out_channels).
void run_to_out(gp_engine* e, Plan* p, int first, float* out, int out_on_host, int out_channels, cudaStream_t s) {
  // eager launches write the result straight into a device `out`; a captured graph has the plan's own buffer baked in
  int& eager_runs = p->eager_runs[first];
  const bool graph_now = uses_graph(e, p) && eager_runs > 0;
  ResultTo result(p, (graph_now || out_on_host) ? p->out_f32 : out);
  if (graph_now) {
    const auto key = std::make_pair(first, out_channels);
    auto it = p->graphs.find(key);
    if (it == p->graphs.end())
      it = p->graphs.emplace(key, capture_graph([&](cudaStream_t cs) { return run_ops(p, first, GP_STAGE_READOUT, out_channels, cs); }))
               .first;
    GP_CUDA(cudaGraphLaunch(it->second, s));
  } else {
    GP_CUDA(run_ops(p, first, GP_STAGE_READOUT, out_channels, s));
    eager_runs++;
  }
  result.deliver(out, out_on_host, out_channels, s);
}

// gp_infer_steps from the encode to the readout (genpercept_pipeline.py:416-472), on the plan's fixed buffers: the staged
// rgb, the noise in out_f32 (when `noise`), and the first n_steps rows of the engine's step tables.  The same launches run
// eagerly or under capture.
cudaError_t run_steps(gp_engine* e, Plan* p, int n_steps, bool noise, int out_channels, cudaStream_t s) {
#define GP_STEP_TRY(call) do { const cudaError_t r__ = (call); if (r__ != cudaSuccess) return r__; } while (0)
  const WeightStore& ws = e->ws;
  const StepTables& st = e->steps;
  GP_STEP_TRY(run_ops(p, GP_STAGE_VAE_ENCODE, GP_STAGE_VAE_ENCODE, out_channels, s));   // rgb_latent (:416)
  const T4& lat = p->rgb_latent;
  const long long npx = lat.pixels();
  uint8_t* A = p->arena;
  void* smp = A + p->sample.off;
  if (noise)                  // marigold: pred_latent = randn (:418-425; the caller draws it with its generator)
    GP_STEP_TRY(nchw4_affine_to_nhwc8(p->out_f32, smp, lat.N, lat.H, lat.W, 1.0f, nullptr, nullptr, ws.bf16, s, ws.split));
  else                        // rgb_blending: pred_latent = rgb_latent (:426-427)
    GP_STEP_TRY(cudaMemcpyAsync(smp, A + lat.off, lat.bytes(), cudaMemcpyDeviceToDevice, s));
  for (int i = 0; i < n_steps; ++i) {                                                   // :443-463
    const float* row = st.table + (size_t)i * st.row;
    GP_STEP_TRY(bias_scatter(row, st.segs, (int)st.host_segs.size(), s));
    GP_STEP_TRY(latent_pack(A + lat.off, smp, A + p->xin.off, npx, e->unet_in_ch, ws.bf16, s, ws.split));
    GP_STEP_TRY(run_ops(p, GP_STAGE_UNET, GP_STAGE_UNET, out_channels, s));
    GP_STEP_TRY(ddim_step(A + p->noise_pred.off, smp, A + p->x0.off, npx, row + st.nbias, ws.bf16, s, ws.split));
  }
  // pred_latent = step_output.pred_original_sample (:465); decode_pred (:507-526); clip + shift in the last kernel
  GP_STEP_TRY(latent_affine(A + p->x0.off, A + p->z.off, npx, 1.0f / kLatentScale, ws.pq_dev, ws.pq_dev + 16, ws.bf16, s,
                            ws.split));
  GP_STEP_TRY(run_ops(p, GP_STAGE_READOUT, GP_STAGE_READOUT, out_channels, s));
  return cudaSuccess;
#undef GP_STEP_TRY
}

// gp_encode and gp_encode_exact: the VAE encoder on the caller's rgb; the latent leaves as fp32 [B,4,h,w], or with
// `pair` as the high-precision mode's (hi, lo) pair, fp32 [B,8,h,w].
gp_status encode(gp_engine* e, const void* rgb, int rgb_dtype, int rgb_on_host, float* latent_dev, void* stream, bool pair) {
  return guarded(e, [&]() {
    const char* fn = pair ? "gp_encode_exact" : "gp_encode";
    Plan* p = current_plan(e, fn);
    GP_REQUIRE(rgb && latent_dev, std::string(fn) + ": bad arguments");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    GP_CUDA(cudaSetDevice(e->cfg.device));
    ArenaUse use(p, s);
    stage_rgb(e, p, rgb, rgb_dtype, rgb_on_host, s, fn);
    GP_CUDA(run_ops(p, GP_STAGE_VAE_ENCODE, GP_STAGE_VAE_ENCODE, 1, s));
    const T4& l = p->rgb_latent;
    if (pair) GP_CUDA(latent_pair_to_nchw(p->arena + l.off, latent_dev, l.N, l.H, l.W, e->ws.bf16, s));
    else GP_CUDA(nhwc8_to_nchw_f32(p->arena + l.off, latent_dev, l.N, l.H, l.W, 4, e->ws.bf16, s, e->ws.split));
    if (rgb_on_host) GP_CUDA(cudaStreamSynchronize(s));
  });
}

// The arena tensor gp_tensor_shape / gp_read_tensor / gp_write_tensor name, and the channels they expose.
const T4& named_tensor(const Plan* p, const char* name, int* creal) {
  const std::map<std::string, std::pair<const T4*, int>> named = {
      {"rgb", {&p->rgb, 3}}, {"rgb_latent", {&p->rgb_latent, 4}}, {"z", {&p->z, 4}}, {"xin", {&p->xin, 8}},
      {"sample", {&p->sample, 4}}, {"noise_pred", {&p->noise_pred, 4}}, {"x0", {&p->x0, 4}},
      {"feat0", {&p->feat[0], p->feat[0].C}}, {"feat1", {&p->feat[1], p->feat[1].C}},
      {"feat2", {&p->feat[2], p->feat[2].C}}, {"feat3", {&p->feat[3], p->feat[3].C}}};
  auto it = named.find(name);
  GP_REQUIRE(it != named.end() && is_set(*it->second.first), std::string("unknown tensor ") + name);
  *creal = it->second.second;
  return *it->second.first;
}

}  // namespace

extern "C" {

gp_status gp_create(const gp_config* cfg, gp_engine** out) {
  return guarded_call([&]() {
    GP_REQUIRE(cfg && out, "gp_create: null config or output pointer");
    *out = nullptr;
    GP_REQUIRE(cfg->dtype == GP_F16 || cfg->dtype == GP_BF16, "gp_create: dtype must be GP_F16 or GP_BF16");
    int ndev = 0;
    GP_CUDA(cudaGetDeviceCount(&ndev));
    const std::string dev = std::to_string(cfg->device);
    if (ndev <= cfg->device)
      throw GpError(GP_ERR_CUDA, "gp_create: no CUDA device " + dev + " (" + std::to_string(ndev) + " visible)");
    GP_CUDA(cudaSetDevice(cfg->device));
    cudaDeviceProp prop;
    GP_CUDA(cudaGetDeviceProperties(&prop, cfg->device));
    if (prop.major != 9)
      throw GpError(GP_ERR_CUDA, "gp_create: device " + dev + " is sm_" + std::to_string(prop.major * 10 + prop.minor) +
                                     "; this library runs on sm_90a only");
    GP_REQUIRE(cfg->arch == 0 || cfg->arch == 1, "gp_create: arch must be 0 (one-step) or 1 (multi-step)");
    GP_REQUIRE(cfg->precision == 0 || cfg->precision == 1, "gp_create: precision must be 0 (default) or 1 (high)");
    gp_engine* e = new gp_engine();   // nothing below throws
    e->cfg = *cfg;
    if (e->cfg.timestep <= 0) e->cfg.timestep = 1;
    e->ws.bf16 = cfg->dtype == GP_BF16;
    e->ws.split = cfg->precision == 1;
    e->multistep = cfg->arch == 1;
    *out = e;
  });
}

void gp_destroy(gp_engine* e) { delete e; }

const char* gp_last_error(gp_engine* e) { return e ? e->err.c_str() : "null engine"; }

const char* gp_last_call_error(void) { return call_error().c_str(); }

gp_status gp_load_tensor(gp_engine* e, const char* key, const void* host_ptr, int dtype, const int64_t* shape, int ndim) {
  return guarded(e, [&]() {
    GP_REQUIRE(key && host_ptr && shape && ndim >= 1 && ndim <= 4, "gp_load_tensor: bad arguments");
    if (e->finalized) throw GpError(GP_ERR_STATE, "gp_load_tensor after gp_finalize");
    const bool text = std::strncmp(key, "text.", 5) == 0;
    if (text) {
      if (std::strcmp(key, "text.text_model.embeddings.position_ids") == 0) return;   // a buffer of arange(77)
      const auto& spec = text_tower_spec();
      auto it = spec.find(key);
      GP_REQUIRE(it != spec.end(), std::string("gp_load_tensor: ") + key + " is not a tensor of SD-2.1's CLIP text tower");
      GP_REQUIRE(std::vector<int64_t>(shape, shape + ndim) == it->second,
                 std::string("gp_load_tensor: ") + key + " does not have the shape of SD-2.1's CLIP text tower (d = 1024, "
                 "23 layers, MLP 4096, vocabulary 49408)");
    }
    HostT t;
    t.shape.assign(shape, shape + ndim);
    const int64_t n = t.numel();
    t.d.resize((size_t)n);
    if (dtype == GP_F32) std::memcpy(t.d.data(), host_ptr, (size_t)n * 4);
    else if (dtype == GP_F16 || dtype == GP_BF16) {
      const uint16_t* s = reinterpret_cast<const uint16_t*>(host_ptr);
      for (int64_t i = 0; i < n; ++i) t.d[(size_t)i] = host_h2f(s[i], dtype == GP_BF16);
    } else throw GpError(GP_ERR_INVALID, "gp_load_tensor: unsupported dtype");
    if (!text) {
      e->ws.host[key] = std::move(t);
      return;
    }
    TextTower& tt = e->text;
    if (!tt.ws || tt.packed) {   // a tensor after gp_encode_text: the next call packs the weights again
      std::unique_ptr<WeightStore> fresh(new WeightStore(e->ws.bf16, e->ws.split));
      if (tt.ws) fresh->host = std::move(tt.ws->host);
      GP_CUDA(cudaSetDevice(e->cfg.device));
      tt.plans.clear();
      tt.ws = std::move(fresh);
      tt.packed = false;
    }
    tt.ws->host[key] = std::move(t);
  });
}

gp_status gp_encode_text(gp_engine* e, const int32_t* ids_host, int n_tokens, float* out_host, void* stream) {
  return guarded(e, [&]() {
    if (e->finalized) throw GpError(GP_ERR_STATE, "gp_encode_text after gp_finalize: the context is a constant of the engine");
    GP_REQUIRE(ids_host && out_host, "gp_encode_text: bad arguments");
    GP_REQUIRE(n_tokens >= 1 && n_tokens <= kTextMaxTokens,
               "gp_encode_text: " + std::to_string(n_tokens) + " tokens (1 to " + std::to_string(kTextMaxTokens) + ")");
    for (int i = 0; i < n_tokens; ++i)
      GP_REQUIRE(ids_host[i] >= 0 && ids_host[i] < kTextVocab,
                 "gp_encode_text: token id " + std::to_string(ids_host[i]) + " outside [0, " + std::to_string(kTextVocab) + ")");
    TextTower& tt = e->text;
    for (const auto& kv : text_tower_spec())
      if (!tt.ws || !tt.ws->host.count(kv.first)) throw GpError(GP_ERR_MISSING, "gp_encode_text: missing " + kv.first);
    GP_CUDA(cudaSetDevice(e->cfg.device));
    TextPlan* p = tt.plan(n_tokens);
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    GP_CUDA(cudaMemcpyAsync(p->ids, ids_host, (size_t)n_tokens * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    for (auto& op : p->ops) GP_CUDA(op.run(s));
    GP_CUDA(cudaMemcpyAsync(out_host, p->out, (size_t)n_tokens * kTextDim * sizeof(float), cudaMemcpyDeviceToHost, s));
    GP_CUDA(cudaStreamSynchronize(s));
  });
}

gp_status gp_set_text_embed(gp_engine* e, const float* host_ptr, int n_tokens, int dim) {
  return guarded(e, [&]() {
    GP_REQUIRE(host_ptr && dim == 1024 && n_tokens >= 1, "gp_set_text_embed: expected [n_tokens, 1024]");
    if (e->finalized) throw GpError(GP_ERR_STATE, "gp_set_text_embed after gp_finalize");
    e->ws.text_embed.assign(host_ptr, host_ptr + (size_t)n_tokens * dim);
    e->ws.n_tokens = n_tokens;
  });
}

gp_status gp_finalize(gp_engine* e) {
  return guarded(e, [&]() {
    if (e->finalized) return;
    GP_REQUIRE(e->ws.n_tokens > 0, "gp_finalize: text embedding not set");
    GP_CUDA(cudaSetDevice(e->cfg.device));
    // A measuring pass over a nominal shape touches every weight the topology needs: packs + uploads.
    Builder b(e->ws.bf16, true, nullptr, e->ws.split);
    e->build(b, nullptr, 1, 64, 64);
    if (e->multistep) e->steps.init(e->ws);
    e->ws.host.clear();
    e->text = TextTower();     // the tower's weights and arenas: gp_encode_text is done once the context is fixed
    e->finalized = true;
  });
}

gp_status gp_plan(gp_engine* e, int B, int H, int W) {
  return guarded(e, [&]() {
    if (!e->finalized) throw GpError(GP_ERR_STATE, "gp_plan before gp_finalize");
    GP_REQUIRE(B >= 1 && H >= 32 && W >= 32, "gp_plan: bad shape (H, W >= 32)");
    GP_CUDA(cudaSetDevice(e->cfg.device));
    auto key = std::make_tuple(B, H, W);
    auto it = e->plans.find(key);
    // Only gp_plan stamps a plan: it is also the only place `cur` changes, so the current plan is always the newest.
    if (it != e->plans.end()) { e->cur = it->second.get(); e->cur->last_used = ++e->use_clock; return; }
    // Bounded plan cache (a folder of in-the-wild images yields a new (H, W) per aspect ratio): evict the least
    // recently used plans — graph execs destroyed, arena freed — before building another one.
    static const size_t max_plans = std::getenv("GP_MAX_PLANS") ? (size_t)std::max(1, std::atoi(std::getenv("GP_MAX_PLANS"))) : 4;
    while (e->plans.size() >= max_plans) {
      auto victim = e->plans.begin();
      for (auto jt = e->plans.begin(); jt != e->plans.end(); ++jt)
        if (jt->second->last_used < victim->second->last_used) victim = jt;
      e->drop_plan(victim);
    }
    Builder m(e->ws.bf16, true, nullptr, e->ws.split);
    m.mem_efficient_attn = e->mem_efficient_attn;
    e->build(m, nullptr, B, H, W);
    std::unique_ptr<Plan> p(new Plan());
    p->B = B; p->H = H; p->W = W;
    p->device = e->cfg.device;
    p->arena_bytes = m.arena_bytes();
    bool too_large = false;
    if (e->shared_arena) {
      p->arena = shared_arena_add(p->device, p->arena_bytes);
      p->shared = p->arena != nullptr;
      too_large = !p->shared;
    } else {
      const cudaError_t ae = cudaMalloc(reinterpret_cast<void**>(&p->arena), p->arena_bytes);
      // Not a sticky error: clear it and report the shape as too large, so the engine stays usable for smaller inputs.
      if (ae == cudaErrorMemoryAllocation) { cudaGetLastError(); too_large = true; }
      else GP_CUDA(ae);
    }
    if (too_large)
      throw GpError(GP_ERR_INVALID, "gp_plan: batch " + std::to_string(B) + " at " + std::to_string(H) + "x" +
                                        std::to_string(W) + " needs an activation arena of " +
                                        std::to_string(p->arena_bytes) + " bytes, more than the device can allocate");
    if (!m.long_softmax.empty()) {
      // The arena fits, but the unfused softmax of this attention cannot run: fail here, not with a CUDA error at
      // inference, and leave the engine usable.
      throw GpError(GP_ERR_INVALID, "gp_plan: batch " + std::to_string(B) + " at " + std::to_string(H) + "x" +
                                        std::to_string(W) + ": " + m.long_softmax + " has rows past " +
                                        std::to_string(kSoftmaxRowsMaxT) + " keys, more than the unfused softmax takes; "
                                        "enable memory-efficient attention (gp_set_memory_efficient_attention)");
    }
    if (p->shared) {   // on the legacy stream like cudaMemset, after the pool's earlier users on any stream
      ArenaUse use(p.get(), nullptr);
      GP_CUDA(cudaMemsetAsync(p->arena, 0, p->arena_bytes, nullptr));
    } else {
      GP_CUDA(cudaMemset(p->arena, 0, p->arena_bytes));
    }
    Builder b(e->ws.bf16, false, p->arena, e->ws.split);
    b.mem_efficient_attn = e->mem_efficient_attn;
    e->build(b, p.get(), B, H, W);
    if (b.arena_bytes() != p->arena_bytes) throw GpError(GP_ERR_STATE, "planner passes disagree on arena size");
    p->ops = std::move(b.ops);
    for (auto& op : p->ops) {
      if (op.variant == 3) continue;
      p->launches += op.launches;
      p->igemm_flops += op.flops;
    }
    p->last_used = ++e->use_clock;
    e->cur = p.get();
    e->plans[key] = std::move(p);
  });
}

int gp_plan_count(gp_engine* e) { return e ? (int)e->plans.size() : 0; }

gp_status gp_set_memory_efficient_attention(gp_engine* e, int enable) {
  return guarded(e, [&]() {
    const bool on = enable != 0;
    if (on == e->mem_efficient_attn) return;
    GP_CUDA(cudaSetDevice(e->cfg.device));
    while (!e->plans.empty()) e->drop_plan(e->plans.begin());
    e->mem_efficient_attn = on;
  });
}

gp_status gp_set_shared_arena(gp_engine* e, int enable) {
  return guarded(e, [&]() {
    const bool on = enable != 0;
    if (on == e->shared_arena) return;
    GP_CUDA(cudaSetDevice(e->cfg.device));
    while (!e->plans.empty()) e->drop_plan(e->plans.begin());
    if (on) shared_arena_join(e->cfg.device);
    else shared_arena_leave(e->cfg.device);
    e->shared_arena = on;
  });
}

gp_status gp_tile_shape(int cout, int cin, int ks, int images, int h, int w, int tokens_mode, int num_sms, int* bn, int* mt) {
  return guarded_call([&]() {
    GP_REQUIRE(bn && mt, "gp_tile_shape: null output pointer");
    GP_REQUIRE(cout >= 1 && cin >= 1 && ks >= 1 && images >= 1 && h >= 1 && w >= 1 && num_sms >= 1,
               "gp_tile_shape: every size must be at least 1");
    gp::tile_shape_for(cout, (double)cin * ks * ks, tokens_mode != 0, images, w, h, num_sms, bn, mt);
  });
}

gp_status gp_conv_tile(int cin, int csc, int cout, int images, int h, int w, int num_sms, int* bn, int* mt, int* patch) {
  return guarded_call([&]() {
    GP_REQUIRE(bn && mt && patch, "gp_conv_tile: null output pointer");
    GP_REQUIRE(cin >= 1 && csc >= 0 && cout >= 1 && images >= 1 && h >= 1 && w >= 1 && num_sms >= 1,
               "gp_conv_tile: every size must be at least 1 (csc at least 0)");
    gp::tile_shape_for(cout, (double)cin * 9 + csc, false, images, w, h, num_sms, bn, mt);
    const bool staged = cout % 64 == 0 && *bn % 64 == 0;   // Builder::conv: the staged epilogue of a 16-bit NHWC output
    *patch = staged && gp::patch_tile_fits(images, h, w, cin, csc, cout, *bn, *mt, num_sms) ? 1 : 0;
  });
}

gp_status gp_step_bias_layout(int capacity, int* n_segments, int* offsets, int* lengths) {
  return guarded_call([&]() {
    GP_REQUIRE(n_segments, "gp_step_bias_layout: null n_segments");
    const auto layout = step_bias_layout();
    *n_segments = (int)layout.size();
    if (capacity < (int)layout.size()) {
      GP_REQUIRE(!offsets && !lengths, "gp_step_bias_layout: capacity " + std::to_string(capacity) + " is below the " +
                                           std::to_string(layout.size()) + " segments");
      return;
    }
    int off = 0;
    for (size_t k = 0; k < layout.size(); ++k) {
      if (offsets) offsets[k] = off;
      if (lengths) lengths[k] = layout[k].second;
      off += layout[k].second;
    }
  });
}

gp_status gp_set_timestep(gp_engine* e, int timestep) {
  return guarded(e, [&]() {
    if (!e->finalized) throw GpError(GP_ERR_STATE, "gp_set_timestep before gp_finalize");
    GP_CUDA(cudaSetDevice(e->cfg.device));
    e->ws.set_timestep(timestep);
  });
}

gp_status gp_infer(gp_engine* e, const void* rgb, int rgb_dtype, int rgb_on_host, float* out, int out_on_host,
                   int out_channels, void* stream) {
  return guarded(e, [&]() {
    Plan* p = current_plan(e, "gp_infer");
    if (e->multistep) throw GpError(GP_ERR_STATE, "gp_infer: this engine runs the multi-step arch (gp_infer_steps)");
    if (e->cfg.readout == GP_READOUT_DPT) out_channels = 1;
    GP_REQUIRE(rgb && out && (out_channels == 1 || out_channels == 3), "gp_infer: bad arguments");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    GP_CUDA(cudaSetDevice(e->cfg.device));
    ArenaUse use(p, s);
    stage_rgb(e, p, rgb, rgb_dtype, rgb_on_host, s, "gp_infer");
    run_to_out(e, p, GP_STAGE_VAE_ENCODE, out, out_on_host, out_channels, s);
    if (rgb_on_host || out_on_host) GP_CUDA(cudaStreamSynchronize(s));
  });
}

gp_status gp_infer_latent(gp_engine* e, const float* latent_dev, int batch, int channels, int height, int width, float* out,
                          int out_on_host, int out_channels, void* stream) {
  return guarded(e, [&]() {
    if (e->multistep) throw GpError(GP_ERR_INVALID, "gp_infer_latent: runs the one-step arch only (gp_config.arch = 0)");
    Plan* p = current_plan(e, "gp_infer_latent");
    if (e->cfg.readout == GP_READOUT_DPT) out_channels = 1;
    GP_REQUIRE(latent_dev && out && (out_channels == 1 || out_channels == 3), "gp_infer_latent: bad arguments");
    const T4& lat = p->rgb_latent;
    const int lat_c = e->ws.split ? 8 : 4;
    GP_REQUIRE(batch == lat.N && channels == lat_c && height == lat.H && width == lat.W,
               "gp_infer_latent: latent [" + std::to_string(batch) + "," + std::to_string(channels) + "," + std::to_string(height) +
                   "," + std::to_string(width) + "] does not match the plan's [" + std::to_string(lat.N) + "," +
                   std::to_string(lat_c) + "," + std::to_string(lat.H) + "," + std::to_string(lat.W) + "]" +
                   (e->ws.split ? " (the high-precision mode takes the (hi, lo) pair gp_encode_exact writes)" : ""));
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    GP_CUDA(cudaSetDevice(e->cfg.device));
    ArenaUse use(p, s);
    if (e->ws.split) GP_CUDA(latent_pair_from_nchw(latent_dev, p->arena + lat.off, lat.N, lat.H, lat.W, e->ws.bf16, s));
    else GP_CUDA(nchw4_affine_to_nhwc8(latent_dev, p->arena + lat.off, lat.N, lat.H, lat.W, 1.0f, nullptr, nullptr, e->ws.bf16, s));
    run_to_out(e, p, GP_STAGE_UNET, out, out_on_host, out_channels, s);
    if (out_on_host) GP_CUDA(cudaStreamSynchronize(s));
  });
}

gp_status gp_encode(gp_engine* e, const void* rgb, int rgb_dtype, int rgb_on_host, float* latent_dev, void* stream) {
  return encode(e, rgb, rgb_dtype, rgb_on_host, latent_dev, stream, false);
}

gp_status gp_encode_exact(gp_engine* e, const void* rgb, int rgb_dtype, int rgb_on_host, float* latent_dev, void* stream) {
  return encode(e, rgb, rgb_dtype, rgb_on_host, latent_dev, stream, e && e->ws.split);
}

gp_status gp_decode(gp_engine* e, const float* latent_dev, int apply_post_quant, float* out_dev, int out_channels, void* stream) {
  return guarded(e, [&]() {
    Plan* p = current_plan(e, "gp_decode");
    if (e->cfg.readout == GP_READOUT_DPT) throw GpError(GP_ERR_STATE, "gp_decode: the DPT readout has no latent decoder");
    GP_REQUIRE(latent_dev && out_dev && (out_channels == 1 || out_channels == 3), "gp_decode: bad arguments");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    GP_CUDA(cudaSetDevice(e->cfg.device));
    ArenaUse use(p, s);
    const T4& z = p->z;
    GP_CUDA(nchw4_affine_to_nhwc8(latent_dev, p->arena + z.off, z.N, z.H, z.W, 1.0f / kLatentScale,
                                  apply_post_quant ? e->ws.pq_dev : nullptr, apply_post_quant ? e->ws.pq_dev + 16 : nullptr, e->ws.bf16, s,
                                  e->ws.split));
    ResultTo result(p, out_dev);
    GP_CUDA(run_ops(p, GP_STAGE_READOUT, GP_STAGE_READOUT, out_channels, s));
  });
}

gp_status gp_infer_steps(gp_engine* e, const void* rgb, int rgb_dtype, int rgb_on_host, const float* noise, int noise_on_host,
                         const int* timesteps, const float* coeffs, int n_steps, float* out, int out_on_host, int out_channels,
                         void* stream) {
  return guarded(e, [&]() {
    Plan* p = current_plan(e, "gp_infer_steps");
    if (!e->multistep) throw GpError(GP_ERR_STATE, "gp_infer_steps needs gp_config.arch = 1");
    GP_REQUIRE(rgb && out && timesteps && coeffs && n_steps >= 1 && (out_channels == 1 || out_channels == 3), "gp_infer_steps: bad arguments");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    GP_CUDA(cudaSetDevice(e->cfg.device));
    ArenaUse use(p, s);
    StepTables& st = e->steps;
    e->reserve_steps(n_steps);
    // Fold this call's rows on the host.  The staging buffer is rewritten only after the previous upload from it is done.
    GP_CUDA(cudaEventSynchronize(st.staged));
    for (int i = 0; i < n_steps; ++i) {
      float* row = st.staging + (size_t)i * st.row;
      for (size_t k = 0; k < st.keys.size(); ++k) {
        const std::vector<float>& b = e->ws.temb_bias(timesteps[i], st.keys[k]);
        std::memcpy(row + st.host_segs[k].off, b.data(), (size_t)st.host_segs[k].len * sizeof(float));
      }
      std::memcpy(row + st.nbias, coeffs + 4 * i, 4 * sizeof(float));
    }
    // The previous call, on whatever stream, is done with the table, the bias buffers and out_f32 before these land.
    GP_CUDA(cudaStreamWaitEvent(s, st.released, 0));
    GP_CUDA(cudaMemcpyAsync(st.table, st.staging, (size_t)n_steps * st.row * sizeof(float), cudaMemcpyHostToDevice, s));
    GP_CUDA(cudaEventRecord(st.staged, s));
    stage_rgb(e, p, rgb, rgb_dtype, rgb_on_host, s, "gp_infer_steps");
    // The caller's noise goes to a fixed buffer, which a graph can read: the plan's result buffer is free until the
    // decoder runs.
    if (noise)
      GP_CUDA(cudaMemcpyAsync(p->out_f32, noise, (size_t)p->rgb_latent.pixels() * 4 * sizeof(float),
                              noise_on_host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, s));
    // As run_to_out: the first pass of a key runs eagerly, later ones replay its graph, which writes out_f32.
    const auto key = std::make_tuple(n_steps, noise ? 1 : 0, out_channels);
    int& eager_runs = p->step_eager_runs[key];
    const bool graph_now = uses_graph(e, p) && eager_runs > 0;
    ResultTo result(p, (graph_now || out_on_host) ? p->out_f32 : out);
    if (graph_now) {
      auto it = p->step_graphs.find(key);
      if (it == p->step_graphs.end())
        it = p->step_graphs
                 .emplace(key, capture_graph([&](cudaStream_t cs) { return run_steps(e, p, n_steps, noise != nullptr, out_channels, cs); }))
                 .first;
      GP_CUDA(cudaGraphLaunch(it->second, s));
    } else {
      GP_CUDA(run_steps(e, p, n_steps, noise != nullptr, out_channels, s));
      eager_runs++;
    }
    e->ws.cur_timestep = timesteps[n_steps - 1];     // the bias buffers hold the last step's values
    result.deliver(out, out_on_host, out_channels, s);
    GP_CUDA(cudaEventRecord(st.released, s));
    if (rgb_on_host || out_on_host) GP_CUDA(cudaStreamSynchronize(s));
  });
}

gp_status gp_run_stage(gp_engine* e, int stage, int out_channels, void* stream) {
  return guarded(e, [&]() {
    Plan* p = current_plan(e, "gp_run_stage");
    if (e->cfg.readout == GP_READOUT_DPT) out_channels = 1;
    GP_CUDA(cudaSetDevice(e->cfg.device));
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    ArenaUse use(p, s);
    ResultTo result(p, p->out_f32);
    GP_CUDA(run_ops(p, stage, stage, out_channels, s));
  });
}

gp_status gp_tensor_shape(gp_engine* e, const char* name, int64_t shape[4]) {
  return guarded(e, [&]() {
    Plan* p = current_plan(e, "gp_tensor_shape");
    if (std::string(name) == "out") { shape[0] = p->B; shape[1] = 3; shape[2] = p->outH; shape[3] = p->outW; return; }
    int cr = 0;
    const T4& t = named_tensor(p, name, &cr);
    shape[0] = t.N; shape[1] = cr; shape[2] = t.H; shape[3] = t.W;
  });
}

gp_status gp_read_tensor(gp_engine* e, const char* name, float* host_out, size_t cap) {
  return guarded(e, [&]() {
    Plan* p = current_plan(e, "gp_read_tensor");
    GP_CUDA(cudaSetDevice(e->cfg.device));
    ArenaUse use(p, nullptr);
    GP_CUDA(cudaDeviceSynchronize());
    if (std::string(name) == "out") {
      const size_t n = (size_t)p->B * 3 * p->outH * p->outW;
      GP_REQUIRE(cap >= n, "gp_read_tensor: buffer too small");
      GP_CUDA(cudaMemcpy(host_out, p->out_f32, n * 4, cudaMemcpyDeviceToHost));
      return;
    }
    int cr = 0;
    const T4& t = named_tensor(p, name, &cr);
    GP_REQUIRE(cap >= (size_t)t.N * cr * t.H * t.W, "gp_read_tensor: buffer too small");
    const size_t ps = (size_t)t.ps();
    std::vector<uint16_t> h((size_t)t.N * t.H * t.W * ps);
    GP_CUDA(cudaMemcpy(h.data(), p->arena + t.off, h.size() * 2, cudaMemcpyDeviceToHost));
    const size_t HW = (size_t)t.H * t.W;
    for (int n = 0; n < t.N; ++n)
      for (size_t px = 0; px < HW; ++px)
        for (int c = 0; c < cr; ++c) {
          const uint16_t* q = &h[((size_t)n * HW + px) * ps + c];
          host_out[((size_t)n * cr + c) * HW + px] = host_h2f(q[0], e->ws.bf16) + (t.planes == 2 ? host_h2f(q[t.C], e->ws.bf16) : 0.f);
        }
  });
}

gp_status gp_write_tensor(gp_engine* e, const char* name, const float* host_in, size_t elems) {
  return guarded(e, [&]() {
    Plan* p = current_plan(e, "gp_write_tensor");
    int cr = 0;
    const T4& t = named_tensor(p, name, &cr);
    GP_REQUIRE(elems == (size_t)t.N * cr * t.H * t.W, "gp_write_tensor: size mismatch");
    const size_t ps = (size_t)t.ps();
    std::vector<uint16_t> h((size_t)t.N * t.H * t.W * ps, 0);
    const size_t HW = (size_t)t.H * t.W;
    for (int n = 0; n < t.N; ++n)
      for (size_t px = 0; px < HW; ++px)
        for (int c = 0; c < cr; ++c) {
          const float v = host_in[((size_t)n * cr + c) * HW + px];
          uint16_t* q = &h[((size_t)n * HW + px) * ps + c];
          q[0] = host_f2h(v, e->ws.bf16);
          if (t.planes == 2) q[t.C] = host_f2h(v - host_h2f(q[0], e->ws.bf16), e->ws.bf16);
        }
    GP_CUDA(cudaSetDevice(e->cfg.device));
    ArenaUse use(p, nullptr);   // the copy may still be in flight when it returns: later users wait for it
    GP_CUDA(cudaDeviceSynchronize());
    GP_CUDA(cudaMemcpy(p->arena + t.off, h.data(), h.size() * 2, cudaMemcpyHostToDevice));
  });
}

gp_status gp_plan_info(gp_engine* e, int64_t* n_ops, int64_t* n_launches, int64_t* arena_bytes, int64_t* weight_bytes,
                       double* igemm_flops) {
  return guarded(e, [&]() {
    Plan* p = current_plan(e, "gp_plan_info");
    if (n_ops) *n_ops = (int64_t)p->ops.size();
    if (n_launches) *n_launches = p->launches + 1;   // + preprocess
    if (arena_bytes) *arena_bytes = (int64_t)p->arena_bytes;
    if (weight_bytes) *weight_bytes = (int64_t)e->ws.weight_bytes;
    if (igemm_flops) *igemm_flops = p->igemm_flops;
  });
}

gp_status gp_profile_ops(gp_engine* e, int out_channels, void* stream) {
  return guarded(e, [&]() {
    Plan* p = current_plan(e, "gp_profile_ops");
    if (e->cfg.readout == GP_READOUT_DPT) out_channels = 1;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    ArenaUse use(p, s);
    cudaEvent_t a, b;
    GP_CUDA(cudaEventCreate(&a));
    GP_CUDA(cudaEventCreate(&b));
    ResultTo result(p, p->out_f32);
    for (auto& op : p->ops) {
      op.usec = 0;
      if (op.variant != 0 && op.variant != out_channels) continue;
      GP_CUDA(cudaEventRecord(a, s));
      GP_CUDA(op.run(s));
      GP_CUDA(cudaEventRecord(b, s));
      GP_CUDA(cudaEventSynchronize(b));
      float ms = 0;
      GP_CUDA(cudaEventElapsedTime(&ms, a, b));
      op.usec = ms * 1000.f;
    }
    cudaEventDestroy(a);
    cudaEventDestroy(b);
  });
}

gp_status gp_op_info(gp_engine* e, int64_t i, char* name_buf, size_t name_cap, double* usec, double* flops, double* bytes,
                     int* kind, double* flops_exec) {
  return guarded(e, [&]() {
    Plan* p = current_plan(e, "gp_op_info");
    GP_REQUIRE(i >= 0 && i < (int64_t)p->ops.size(), "op index out of range");
    const Op& op = p->ops[(size_t)i];
    if (name_buf && name_cap) { std::strncpy(name_buf, op.name.c_str(), name_cap - 1); name_buf[name_cap - 1] = 0; }
    if (usec) *usec = op.usec;
    if (flops) *flops = op.flops;
    if (bytes) *bytes = op.bytes;
    if (kind) *kind = op.kind;
    if (flops_exec) *flops_exec = op.flops_exec >= 0 ? op.flops_exec : op.flops;
  });
}

}  // extern "C"
