// The engine: checkpoint store, constant folding + weight packing (SURVEY.md App. C), the SD-2.1
// GenPercept graph (VAE encoder -> UNet(t, empty-text) -> VAE decoder | DPT head) expressed on the
// Builder, plan cache, CUDA-graph execution and the C-ABI.
//
// Graph semantics follow the reference call sites:
//   /root/reference/genpercept/genpercept_pipeline.py:375-526 (single_infer / encode_rgb / decode_pred)
//   /root/reference/genpercept/models/custom_unet.py:146-170,273,305-327,341-352,369-415
//   /root/reference/genpercept/models/dpt_head.py:52-90,213-335,338-388,530-546,564-592
// and the diffusers block definitions restated in SURVEY.md Appendix A.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <cmath>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <thread>
#include <tuple>

#include "engine.h"

using namespace gp;

namespace {

constexpr float kLatentScale = 0.18215f;   // genpercept_pipeline.py:96
const int kUnetOut[4] = {320, 640, 1280, 1280};
const int kUnetHeads[4] = {5, 10, 20, 20};

int ceil_div_i(int a, int b) { return (a + b - 1) / b; }

uint16_t host_f2h(float f, bool bf16) {
  if (bf16) {
    __nv_bfloat16 h = __float2bfloat16_rn(f);
    uint16_t u;
    std::memcpy(&u, &h, 2);
    return u;
  }
  __half h = __float2half_rn(f);
  uint16_t u;
  std::memcpy(&u, &h, 2);
  return u;
}
float host_h2f(uint16_t u, bool bf16) {
  if (bf16) {
    __nv_bfloat16 h;
    std::memcpy(&h, &u, 2);
    return __bfloat162float(h);
  }
  __half h;
  std::memcpy(&h, &u, 2);
  return __half2float(h);
}

template <class F>
void parallel_for(int n, F f) {
  int nt = (int)std::thread::hardware_concurrency();
  if (nt < 1) nt = 1;
  if (nt > 16) nt = 16;
  if (nt > n) nt = n;
  if (nt <= 1) { for (int i = 0; i < n; ++i) f(i); return; }
  std::vector<std::thread> th;
  for (int t = 0; t < nt; ++t)
    th.emplace_back([=]() { for (int i = t; i < n; i += nt) f(i); });
  for (auto& x : th) x.join();
}

struct Kept {
  T4 t;                 // 16-bit NHWC tensor ...
  float* f32 = nullptr; // ... or fp32 NCHW buffer [N, C, H, W]
  int creal = 0;        // channels exposed through read/write
};

struct Plan {
  int B = 0, H = 0, W = 0;
  uint8_t* arena = nullptr;
  size_t arena_bytes = 0;
  std::vector<Op> ops;
  std::map<std::string, Kept> kept;
  void* in_staging = nullptr;       // raw user input copy [B,3,H,W] (<= 4 bytes/elt), host inputs only
  float* out_f32 = nullptr;         // [B,3,outH,outW]: the plan's own result buffer (graph replay, host outputs, stage runs)
  float* out_dst = nullptr;         // where the final kernels write THIS launch (the caller's device buffer or out_f32);
                                    // read by the ops at launch time through Builder::out_slot
  int outH = 0, outW = 0;           // result extent: 8 * floor(H/8) (VAE readout), 64 * ceil-pyramid (DPT readout)
  uint64_t last_used = 0;
  std::map<int, cudaGraphExec_t> graphs;   // by out_channels
  double igemm_flops = 0;
  int eager_runs = 0;                       // the first pass runs eagerly (kernel attributes, lazy init), then graphs
  int64_t launches = 0;
};

}  // namespace

struct gp_engine {
  gp_config cfg;
  bool bf16 = false;
  bool split = false;        // cfg.precision == 1: (hi, lo) fp16 pairs everywhere (engine.h T4::planes, PackedW::planes)
  std::string err;
  bool poisoned = false, finalized = false;
  std::unordered_map<std::string, HostT> host;
  std::vector<float> text_embed;
  int n_tokens = 0;
  std::unordered_map<std::string, PackedW> packed;
  std::unordered_map<std::string, NormW> norms;
  std::unordered_map<std::string, XattnW> xattns;
  std::unordered_map<std::string, DirectW> directs;
  std::vector<void*> dev_allocs;
  size_t weight_bytes = 0;
  float* pq_dev = nullptr;   // vae.post_quant_conv: [16] weight + [4] bias, fp32 on the device
  bool multistep = false;    // cfg.arch == 1: real DDIM steps around the UNet (SURVEY.md §8 f4), no scheduler fold
  int unet_in_ch = 0;        // 4, or 8 for the marigold arch (cat([rgb_latent, pred_latent]))
  std::vector<float> temb;   // [1280] time embedding for the current timestep
  // Per-call fix_timesteps (genpercept_pipeline.py:405-408): the timestep only enters through
  // conv1.bias + time_emb_proj(silu(emb(t))) of the 22 UNet ResNets, so changing it re-folds those biases in place
  // (the device bias buffers keep their addresses: every plan and captured graph sees the new values).
  struct TembLayer { std::string key; std::vector<float> w, b, conv_bias; float* dev_bias = nullptr; int cout = 0; };
  std::vector<TembLayer> temb_layers;
  std::vector<float> te_w1, te_b1, te_w2, te_b2;
  std::map<int, std::vector<std::vector<float>>> temb_cache;   // timestep -> folded bias per layer
  int cur_timestep = 0;
  uint64_t use_clock = 0;
  std::map<std::tuple<int, int, int>, std::unique_ptr<Plan>> plans;
  Plan* cur = nullptr;

  // ------------------------------------------------------------------ host tensor access
  const HostT& T(const std::string& k) const {
    auto it = host.find(k);
    if (it == host.end()) throw GpError(GP_ERR_MISSING, "missing checkpoint tensor: " + k);
    return it->second;
  }
  bool has(const std::string& k) const { return host.count(k) != 0; }

  template <class Tp>
  Tp* upload(const std::vector<Tp>& v) {
    void* d = nullptr;
    GP_CUDA(cudaMalloc(&d, std::max<size_t>(v.size() * sizeof(Tp), 16)));
    GP_CUDA(cudaMemcpy(d, v.data(), v.size() * sizeof(Tp), cudaMemcpyHostToDevice));
    dev_allocs.push_back(d);
    weight_bytes += v.size() * sizeof(Tp);
    return reinterpret_cast<Tp*>(d);
  }

  // ------------------------------------------------------------------ packing
  // [nz][rows][ktot] 16-bit K-major; each segment padded to a multiple of 64 channels.
  PackedW pack(const std::vector<std::vector<SegSpec>>& classes, int rows, const std::vector<float>& bias) {
    PackedW w;
    w.rows = rows;
    w.nz = (int)classes.size();
    int ktot = 0;
    for (auto& s : classes[0]) ktot += ceil_div_i(s.C, 64) * 64;
    w.ktot = ktot;
    w.planes = split ? 2 : 1;
    const size_t rowlen = (size_t)ktot * w.planes;       // [ktot hi | ktot lo]
    std::vector<uint16_t> buf((size_t)w.nz * rows * rowlen, 0);
    const bool bf = bf16, sp = split;
    for (int z = 0; z < w.nz; ++z) {
      const auto& segs = classes[z];
      uint16_t* base = buf.data() + (size_t)z * rows * rowlen;
      parallel_for(rows, [&, base](int co) {
        uint16_t* row = base + (size_t)co * rowlen;
        int k0 = 0;
        for (auto& sg : segs) {
          for (int c = 0; c < sg.C; ++c) {
            float v = 0.f;
            for (auto& t : sg.terms) v += t.coef * t.p[co * t.sco + c * t.sc];
            const uint16_t hi = host_f2h(v, bf);
            row[k0 + c] = hi;
            if (sp) row[ktot + k0 + c] = host_f2h(v - host_h2f(hi, bf), bf);
          }
          k0 += ceil_div_i(sg.C, 64) * 64;
        }
      });
    }
    w.w = upload(buf);
    if (!bias.empty()) {
      GP_REQUIRE((int)bias.size() == rows, "bias size mismatch");
      std::vector<float> b = bias;
      b.resize(ceil_div_i(rows, 32) * 32 + 32, 0.f);   // float4 loads may run into the padding
      w.bias = upload(b);
    }
    return w;
  }

  // 3x3 (or 1x1) convolution weights, tap-major, sources concatenated; optional fused 1x1 shortcut
  const PackedW& conv_w(const std::string& key, const std::vector<int>& srcC, const std::string& sc_key = "",
                        const std::vector<int>& scC = {}, const std::vector<float>* extra_bias = nullptr,
                        bool want_bias = true, const std::string& cache_suffix = "") {
    auto it = packed.find(key + cache_suffix);
    if (it != packed.end()) return it->second;
    const HostT& w = T(key + ".weight");
    GP_REQUIRE(w.shape.size() == 4, key + ": conv weight must be 4-D");
    const int cout = (int)w.shape[0], cin = (int)w.shape[1], ks = (int)w.shape[2];
    int sum = 0;
    for (int c : srcC) sum += c;
    GP_REQUIRE(sum == cin, key + ": source channels != Cin");
    std::vector<SegSpec> segs;
    for (int r = 0; r < ks; ++r)
      for (int s = 0; s < ks; ++s) {
        int c0 = 0;
        for (int c : srcC) {
          SegSpec sg;
          sg.C = c;
          sg.terms.push_back(Term{w.d.data() + (long long)c0 * ks * ks + r * ks + s, (long long)cin * ks * ks, ks * ks, 1.f});
          segs.push_back(sg);
          c0 += c;
        }
      }
    std::vector<float> bias(cout, 0.f);
    if (want_bias && has(key + ".bias")) bias = T(key + ".bias").d;
    if (!sc_key.empty()) {
      const HostT& ws = T(sc_key + ".weight");
      const int scin = (int)ws.shape[1];
      int c0 = 0;
      for (int c : scC) {
        SegSpec sg;
        sg.C = c;
        sg.terms.push_back(Term{ws.d.data() + c0, (long long)scin, 1, 1.f});
        segs.push_back(sg);
        c0 += c;
      }
      GP_REQUIRE(c0 == scin, sc_key + ": shortcut channels mismatch");
      const HostT& bs = T(sc_key + ".bias");
      for (int i = 0; i < cout; ++i) bias[i] += bs.d[i];
    }
    if (extra_bias)
      for (int i = 0; i < cout; ++i) bias[i] += (*extra_bias)[i];
    return packed.emplace(key + cache_suffix, pack({segs}, cout, bias)).first->second;
  }

  // nearest-2x upsample followed by 3x3 conv == four parity-specific 2x2 convs on the source grid
  const PackedW& conv_up_w(const std::string& key) {
    auto it = packed.find(key);
    if (it != packed.end()) return it->second;
    const HostT& w = T(key + ".weight");
    const int cout = (int)w.shape[0], cin = (int)w.shape[1];
    std::vector<std::vector<SegSpec>> classes;
    for (int cls = 0; cls < 4; ++cls) {
      const int py = cls >> 1, px = cls & 1;
      std::vector<SegSpec> segs;
      for (int a = 0; a < 2; ++a)
        for (int b = 0; b < 2; ++b) {
          SegSpec sg;
          sg.C = cin;
          // rows of the 3x3 kernel that land on source row (y2 + py - 1 + a)
          std::vector<int> rs, ss;
          for (int r = 0; r < 3; ++r) if ((int)std::floor((py + r - 1) / 2.0) == py - 1 + a) rs.push_back(r);
          for (int s = 0; s < 3; ++s) if ((int)std::floor((px + s - 1) / 2.0) == px - 1 + b) ss.push_back(s);
          for (int r : rs)
            for (int s : ss)
              sg.terms.push_back(Term{w.d.data() + r * 3 + s, (long long)cin * 9, 9, 1.f});
          segs.push_back(sg);
        }
      classes.push_back(segs);
    }
    return packed.emplace(key, pack(classes, cout, T(key + ".bias").d)).first->second;
  }

  const PackedW& mat_w(const std::string& cache_key, int rows, int K, const float* m, const std::vector<float>& bias) {
    auto it = packed.find(cache_key);
    if (it != packed.end()) return it->second;
    SegSpec sg;
    sg.C = K;
    sg.terms.push_back(Term{m, (long long)K, 1, 1.f});
    return packed.emplace(cache_key, pack({{sg}}, rows, bias)).first->second;
  }
  const PackedW& lin_w(const std::string& key, bool bias = true) {
    auto it = packed.find(key);
    if (it != packed.end()) return it->second;
    const HostT& w = T(key + ".weight");
    const int rows = (int)w.shape[0], K = (int)(w.numel() / rows);   // also accepts 1x1 conv weights
    return mat_w(key, rows, K, w.d.data(), bias ? T(key + ".bias").d : std::vector<float>());
  }
  const NormW& norm_w(const std::string& key) {
    auto it = norms.find(key);
    if (it != norms.end()) return it->second;
    NormW n;
    n.C = (int)T(key + ".weight").d.size();
    n.gamma = upload(T(key + ".weight").d);
    n.beta = upload(T(key + ".bias").d);
    return norms.emplace(key, n).first->second;
  }
  const DirectW& direct_w(const std::string& key, int cin_used, const std::vector<float>* w_override = nullptr,
                          const std::vector<float>* b_override = nullptr, int cout_override = 0) {
    auto it = directs.find(key);
    if (it != directs.end()) return it->second;
    const HostT& w = T(key + ".weight");
    const int cout = cout_override ? cout_override : (int)w.shape[0];
    const int cin = (int)w.shape[1], ks = (int)w.shape[2];
    GP_REQUIRE(cin == cin_used, key + ": direct conv Cin mismatch");
    const std::vector<float>& src = w_override ? *w_override : w.d;
    std::vector<float> t((size_t)ks * ks * cin * cout);
    for (int co = 0; co < cout; ++co)
      for (int ci = 0; ci < cin; ++ci)
        for (int r = 0; r < ks * ks; ++r) t[((size_t)r * cin + ci) * cout + co] = src[((size_t)co * cin + ci) * ks * ks + r];
    DirectW d;
    d.Cin = cin; d.Cout = cout; d.ks = ks;
    d.w = upload(t);
    if (b_override) d.bias = upload(*b_override);
    else if (has(key + ".bias")) d.bias = upload(T(key + ".bias").d);
    return directs.emplace(key, d).first->second;
  }

  // 2-token cross-attention closed form (SURVEY.md F6), LayerNorm affine folded into U / u0
  const XattnW& xattn_w(const std::string& blk /* ...transformer_blocks.0 */, int C, int heads) {
    auto it = xattns.find(blk);
    if (it != xattns.end()) return it->second;
    GP_REQUIRE(n_tokens == 2, "closed-form cross-attention needs the 2-token empty-prompt embedding");
    const int d = C / heads;
    const HostT &wq = T(blk + ".attn2.to_q.weight"), &wk = T(blk + ".attn2.to_k.weight"), &wv = T(blk + ".attn2.to_v.weight");
    const HostT &wo = T(blk + ".attn2.to_out.0.weight"), &bo = T(blk + ".attn2.to_out.0.bias");
    const HostT &g = T(blk + ".norm2.weight"), &b = T(blk + ".norm2.bias");
    const int E = (int)wk.shape[1];
    std::vector<double> K(2 * C), V(2 * C);
    for (int t = 0; t < 2; ++t)
      for (int c = 0; c < C; ++c) {
        double sk = 0, sv = 0;
        for (int e = 0; e < E; ++e) {
          sk += (double)text_embed[t * E + e] * wk.d[(size_t)c * E + e];
          sv += (double)text_embed[t * E + e] * wv.d[(size_t)c * E + e];
        }
        K[t * C + c] = sk; V[t * C + c] = sv;
      }
    const double scale = 1.0 / std::sqrt((double)d);
    std::vector<float> U((size_t)heads * C), u0(heads), M((size_t)heads * C), c0(C);
    for (int h = 0; h < heads; ++h) {
      double acc0 = 0;
      for (int ci = 0; ci < C; ++ci) {
        double s = 0;
        for (int j = 0; j < d; ++j) s += (double)wq.d[(size_t)(h * d + j) * C + ci] * (K[h * d + j] - K[C + h * d + j]);
        s *= scale;
        U[(size_t)h * C + ci] = (float)(s * g.d[ci]);
        acc0 += s * b.d[ci];
      }
      u0[h] = (float)acc0;
      for (int co = 0; co < C; ++co) {
        double s = 0;
        for (int j = 0; j < d; ++j) s += (V[h * d + j] - V[C + h * d + j]) * wo.d[(size_t)co * C + h * d + j];
        M[(size_t)h * C + co] = (float)s;
      }
    }
    for (int co = 0; co < C; ++co) {
      double s = bo.d[co];
      for (int j = 0; j < C; ++j) s += V[C + j] * wo.d[(size_t)co * C + j];
      c0[co] = (float)s;
    }
    XattnW x;
    x.C = C; x.heads = heads;
    x.U = upload(U); x.u0 = upload(u0); x.M = upload(M); x.c0 = upload(c0);
    return xattns.emplace(blk, x).first->second;
  }

  // General cross-attention over a constant n-token context (non-empty prompts, SURVEY.md §8 f3).  Both projections of
  // the context are constants of the pipeline, so per head h
  //     scores_h = LN(x) A_h,   A_h = Wq_h^T K_h^T / sqrt(d)   ([C] -> [n]),   K = ctx Wk^T
  //     out     += P_h B_h,     B_h = V_h Wo_h^T               ([n] -> [C]),   V = ctx Wv^T
  // i.e. two 1x1 GEMMs ([C] -> [heads*n] and back, columns padded to a multiple of 64) around a per-head softmax.
  struct XattnGen { const PackedW* A; const PackedW* B; int Kp; };
  std::unordered_map<std::string, XattnGen> xattn_gens;
  const XattnGen& xattn_general_w(const std::string& blk, int C, int heads) {
    auto it = xattn_gens.find(blk);
    if (it != xattn_gens.end()) return it->second;
    const int n = n_tokens, d = C / heads;
    const int Kp = (heads * n + 63) / 64 * 64;
    XattnGen xg;
    xg.Kp = Kp;
    if (!packed.count(blk + ".attn2.A")) {
      const HostT &wq = T(blk + ".attn2.to_q.weight"), &wk = T(blk + ".attn2.to_k.weight"), &wv = T(blk + ".attn2.to_v.weight");
      const HostT &wo = T(blk + ".attn2.to_out.0.weight"), &bo = T(blk + ".attn2.to_out.0.bias");
      const int E = (int)wk.shape[1];
      std::vector<float> K((size_t)n * C), V((size_t)n * C);
      for (int t = 0; t < n; ++t)
        for (int c = 0; c < C; ++c) {
          double sk = 0, sv = 0;
          const float* te = &text_embed[(size_t)t * E];
          const float *rk = &wk.d[(size_t)c * E], *rv = &wv.d[(size_t)c * E];
          for (int e = 0; e < E; ++e) { sk += (double)te[e] * rk[e]; sv += (double)te[e] * rv[e]; }
          K[(size_t)t * C + c] = (float)sk; V[(size_t)t * C + c] = (float)sv;
        }
      const double scale = 1.0 / std::sqrt((double)d);
      std::vector<float> A((size_t)Kp * C, 0.f), Bm((size_t)C * Kp, 0.f);
      for (int h = 0; h < heads; ++h)
        for (int j = 0; j < n; ++j) {
          float* row = &A[(size_t)(h * n + j) * C];
          for (int dd = 0; dd < d; ++dd) {
            const float kv = (float)(K[(size_t)j * C + h * d + dd] * scale);
            const float* wr = &wq.d[(size_t)(h * d + dd) * C];
            for (int ci = 0; ci < C; ++ci) row[ci] += wr[ci] * kv;
          }
          for (int co = 0; co < C; ++co) {
            double s = 0;
            const float* wr = &wo.d[(size_t)co * C + h * d];
            const float* vr = &V[(size_t)j * C + h * d];
            for (int dd = 0; dd < d; ++dd) s += (double)wr[dd] * vr[dd];
            Bm[(size_t)co * Kp + h * n + j] = (float)s;
          }
        }
      mat_w(blk + ".attn2.A", Kp, C, A.data(), {});
      mat_w(blk + ".attn2.B", C, Kp, Bm.data(), bo.d);
    }
    xg.A = &packed.at(blk + ".attn2.A");
    xg.B = &packed.at(blk + ".attn2.B");
    return xattn_gens.emplace(blk, xg).first->second;
  }

  void compute_temb() {
    if (!temb.empty()) return;
    if (te_w1.empty()) {
      te_w1 = T("unet.time_embedding.linear_1.weight").d; te_b1 = T("unet.time_embedding.linear_1.bias").d;
      te_w2 = T("unet.time_embedding.linear_2.weight").d; te_b2 = T("unet.time_embedding.linear_2.bias").d;
    }
    temb = temb_for(cfg.timestep);
    cur_timestep = cfg.timestep;
  }
  std::vector<float> temb_for(int timestep) const {
    struct V { const std::vector<float>& d; };
    const V w1{te_w1}, b1{te_b1}, w2{te_w2}, b2{te_b2};
    std::vector<float> e(320), h(1280), temb;
    const float t = (float)timestep;
    for (int i = 0; i < 160; ++i) {   // Timesteps(320, flip_sin_to_cos=True, freq_shift=0), fp32
      const float f = std::exp(-std::log(10000.0f) * (float)i / 160.0f);
      e[i] = std::cos(t * f);
      e[160 + i] = std::sin(t * f);
    }
    for (int o = 0; o < 1280; ++o) {
      double s = b1.d[o];
      for (int i = 0; i < 320; ++i) s += (double)w1.d[(size_t)o * 320 + i] * e[i];
      h[o] = (float)(s / (1.0 + std::exp(-s)));
    }
    temb.assign(1280, 0.f);
    for (int o = 0; o < 1280; ++o) {
      double s = b2.d[o];
      for (int i = 0; i < 1280; ++i) s += (double)w2.d[(size_t)o * 1280 + i] * h[i];
      temb[o] = (float)s;
    }
    return temb;
  }
  static std::vector<float> temb_proj_of(const std::vector<float>& w, const std::vector<float>& b, const std::vector<float>& emb) {
    const int cout = (int)b.size();
    std::vector<double> se(1280);
    for (int i = 0; i < 1280; ++i) se[i] = emb[i] / (1.0 + std::exp(-(double)emb[i]));
    std::vector<float> out(cout);
    for (int o = 0; o < cout; ++o) {
      double s = b[o];
      const float* wr = &w[(size_t)o * 1280];
      for (int i = 0; i < 1280; ++i) s += (double)wr[i] * se[i];
      out[o] = (float)s;
    }
    return out;
  }
  std::vector<float> temb_proj(const std::string& key) {   // time_emb_proj(silu(emb)), SURVEY.md F8
    return temb_proj_of(T(key + ".weight").d, T(key + ".bias").d, temb);
  }

  // ------------------------------------------------------------------ graph pieces
  // 3x3 conv whose input is an NHWC8 tensor with `cin` (4 or 8) real channels: one 64-wide K chunk
  // per tap through the tensor-core kernel (the TMA box zero-fills channels >= 8).
  void small_cin_conv(Builder& b, const std::string& key, const T4& src8, int cin, const T4& out) {
    ConvArgs c;
    c.srcs = {src8};
    c.w = &conv_w(key, {cin});
    c.out = out;
    c.want_stats = true;
    b.conv(key, c);
  }

  T4 resnet(Builder& b, const std::string& p, const std::vector<T4>& xs, int cout, float eps, bool temb_on) {
    int cin = 0;
    std::vector<int> cs;
    for (auto& x : xs) { cin += x.C; cs.push_back(x.C); }
    const T4& x0 = xs[0];
    // norm1 -> SiLU -> conv1 and norm2 -> SiLU -> conv2: the normalisation is an attribute of the convolution (fused into
    // its operand path where the patch-resident kernel applies, materialised by Builder::conv elsewhere)
    T4 h = b.alloc(x0.N, x0.H, x0.W, cout);
    {
      std::vector<float> tp;
      const bool first = temb_on && !packed.count(p + ".conv1");
      if (first) tp = temb_proj(p + ".time_emb_proj");
      ConvArgs c;
      c.srcs = xs;
      c.gn = &norm_w(p + ".norm1"); c.gn_name = p + ".norm1"; c.gn_eps = eps;
      c.w = &conv_w(p + ".conv1", {cin}, "", {}, tp.empty() ? nullptr : &tp);
      if (first) {   // what gp_set_timestep needs to re-fold this bias for another timestep
        TembLayer tl;
        tl.key = p;
        tl.w = T(p + ".time_emb_proj.weight").d;
        tl.b = T(p + ".time_emb_proj.bias").d;
        tl.conv_bias = T(p + ".conv1.bias").d;
        tl.dev_bias = c.w->bias;
        tl.cout = cout;
        temb_layers.push_back(std::move(tl));
      }
      c.out = h;
      c.want_stats = true;     // feeds norm2
      b.conv(p + ".conv1", c);
    }
    T4 out = b.alloc(x0.N, x0.H, x0.W, cout);
    {
      ConvArgs c;
      c.srcs = {h};
      c.gn = &norm_w(p + ".norm2"); c.gn_name = p + ".norm2"; c.gn_eps = eps;
      c.out = out;
      c.want_stats = true;     // resnet outputs feed the next GroupNorm (norm1 / transformer norm / conv_norm_out)
      if (cin != cout) {
        c.sc = xs;
        c.w = &conv_w(p + ".conv2", {cout}, p + ".conv_shortcut", cs);
      } else {
        c.w = &conv_w(p + ".conv2", {cout});
        c.res1 = &xs[0];
      }
      b.conv(p + ".conv2", c);
    }
    b.release(h);
    return out;
  }

  T4 transformer(Builder& b, const std::string& p, const T4& x, int heads) {
    const int C = x.C;
    const std::string blk = p + ".transformer_blocks.0";
    T4 n = b.alloc(x.N, x.H, x.W, C);
    b.gn(p + ".norm", {x}, norm_w(p + ".norm"), 32, 1e-6f, false, n);
    T4 t = b.alloc(x.N, x.H, x.W, C);
    { ConvArgs c; c.srcs = {n}; c.ks = 1; c.w = &lin_w(p + ".proj_in"); c.out = t; b.conv(p + ".proj_in", c); }
    b.release(n);
    // self attention
    T4 l = b.alloc(x.N, x.H, x.W, C);
    b.ln(blk + ".norm1", t, norm_w(blk + ".norm1"), 1e-5f, l);
    if (!packed.count(blk + ".attn1.to_qk")) {
      const HostT &wq = T(blk + ".attn1.to_q.weight"), &wk = T(blk + ".attn1.to_k.weight");
      const float scale = 1.0f / std::sqrt((float)(C / heads));
      std::vector<float> m((size_t)2 * C * C);
      for (size_t i = 0; i < (size_t)C * C; ++i) { m[i] = wq.d[i] * scale; m[(size_t)C * C + i] = wk.d[i]; }
      mat_w(blk + ".attn1.to_qk", 2 * C, C, m.data(), {});
    }
    T4 o = b.alloc(x.N, x.H, x.W, C);
    b.attention(blk + ".attn1", l, packed.at(blk + ".attn1.to_qk"), lin_w(blk + ".attn1.to_v", false), nullptr, heads, o);
    b.release(l);
    T4 t1 = b.alloc(x.N, x.H, x.W, C);
    { ConvArgs c; c.srcs = {o}; c.ks = 1; c.w = &lin_w(blk + ".attn1.to_out.0"); c.out = t1; c.res1 = &t; b.conv(blk + ".attn1.to_out", c); }
    b.release(o);
    b.release(t);
    // cross attention (2-token closed form, fused with its LayerNorm and residual)
    T4 t2 = b.alloc(x.N, x.H, x.W, C);
    if (n_tokens == 2) {
      b.xattn(blk + ".attn2", t1, xattn_w(blk, C, heads), 1e-5f, t2);
    } else {   // general context length: LN -> [C -> heads*n] GEMM -> per-head softmax -> [heads*n -> C] GEMM + residual
      const XattnGen& xg = xattn_general_w(blk, C, heads);
      T4 l2 = b.alloc(x.N, x.H, x.W, C);
      b.ln(blk + ".norm2", t1, norm_w(blk + ".norm2"), 1e-5f, l2);
      T4 sc = b.alloc(x.N, x.H, x.W, xg.Kp);
      { ConvArgs c; c.srcs = {l2}; c.ks = 1; c.w = xg.A; c.out = sc; b.conv(blk + ".attn2.scores", c); }
      b.release(l2);
      if (!b.measuring()) {
        void* sp = b.ptr(sc);
        const long long rows = (long long)x.N * x.H * x.W;
        const int kp = xg.Kp, nh = heads, nt = n_tokens;
        const bool bf = bf16, spl = split;
        b.custom(blk + ".attn2.softmax", 1, 2.0 * rows * kp * 2,
                 [=](cudaStream_t s) { return softmax_groups(sp, rows, kp, nh, nt, bf, s, spl); });
      }
      { ConvArgs c; c.srcs = {sc}; c.ks = 1; c.w = xg.B; c.out = t2; c.res1 = &t1; b.conv(blk + ".attn2.out", c); }
      b.release(sc);
    }
    b.release(t1);
    // feed-forward (GEGLU)
    T4 l3 = b.alloc(x.N, x.H, x.W, C);
    b.ln(blk + ".norm3", t2, norm_w(blk + ".norm3"), 1e-5f, l3);
    // GEGLU fused into the projection's epilogue: weight rows interleaved [16 values | 16 gates] per
    // 32-column chunk so one thread holds a value and its gate; the 8C-wide tensor is never written.
    if (!packed.count(blk + ".ff.geglu_w")) {
      const HostT &w = T(blk + ".ff.net.0.proj.weight"), &bb = T(blk + ".ff.net.0.proj.bias");
      const int C4 = 4 * C;
      std::vector<float> m((size_t)8 * C * C), bias(8 * C);
      for (int r = 0; r < 8 * C; ++r) {
        const int chunk = r / 32, q = r % 32;
        const int src = q < 16 ? chunk * 16 + q : C4 + chunk * 16 + (q - 16);
        std::memcpy(&m[(size_t)r * C], &w.d[(size_t)src * C], (size_t)C * sizeof(float));
        bias[r] = bb.d[src];
      }
      mat_w(blk + ".ff.geglu_w", 8 * C, C, m.data(), bias);
    }
    T4 gg = b.alloc(x.N, x.H, x.W, 4 * C);
    {
      ConvArgs c; c.srcs = {l3}; c.ks = 1; c.w = &packed.at(blk + ".ff.geglu_w"); c.out = gg; c.cout_valid = 8 * C;
      c.flags = IG_GEGLU; c.force_bn = 128;
      b.conv(blk + ".ff.proj_geglu", c);
    }
    b.release(l3);
    T4 t3 = b.alloc(x.N, x.H, x.W, C);
    { ConvArgs c; c.srcs = {gg}; c.ks = 1; c.w = &lin_w(blk + ".ff.net.2"); c.out = t3; c.res1 = &t2; b.conv(blk + ".ff.out", c); }
    b.release(gg);
    b.release(t2);
    T4 out = b.alloc(x.N, x.H, x.W, C);
    { ConvArgs c; c.srcs = {t3}; c.ks = 1; c.w = &lin_w(p + ".proj_out"); c.out = out; c.res1 = &x; c.want_stats = true; b.conv(p + ".proj_out", c); }
    b.release(t3);
    return out;
  }

  T4 vae_mid(Builder& b, const std::string& p, T4 x) {
    T4 r0 = resnet(b, p + ".resnets.0", {x}, 512, 1e-6f, false);
    b.release(x);
    const std::string a = p + ".attentions.0";
    T4 n = b.alloc(r0.N, r0.H, r0.W, 512);
    b.gn(a + ".group_norm", {r0}, norm_w(a + ".group_norm"), 32, 1e-6f, false, n);
    if (!packed.count(a + ".to_qk")) {
      const HostT &wq = T(a + ".to_q.weight"), &wk = T(a + ".to_k.weight"), &bq = T(a + ".to_q.bias"), &bk = T(a + ".to_k.bias");
      const float scale = 1.0f / std::sqrt(512.0f);
      std::vector<float> m((size_t)1024 * 512), bias(1024);
      for (size_t i = 0; i < (size_t)512 * 512; ++i) { m[i] = wq.d[i] * scale; m[(size_t)512 * 512 + i] = wk.d[i]; }
      for (int i = 0; i < 512; ++i) { bias[i] = bq.d[i] * scale; bias[512 + i] = bk.d[i]; }
      mat_w(a + ".to_qk", 1024, 512, m.data(), bias);
    }
    // softmax rows sum to 1 -> the V bias passes through P.V unchanged: add it in the PV epilogue
    if (!norms.count(a + ".to_v.biasbuf")) {
      NormW nb;
      std::vector<float> bv = T(a + ".to_v.bias").d;
      bv.resize(512 + 64, 0.f);
      nb.gamma = upload(bv);
      nb.C = 512;
      norms.emplace(a + ".to_v.biasbuf", nb);
    }
    T4 o = b.alloc(r0.N, r0.H, r0.W, 512);
    b.attention(a, n, packed.at(a + ".to_qk"), lin_w(a + ".to_v", false), norms.at(a + ".to_v.biasbuf").gamma, 1, o);
    b.release(n);
    T4 y = b.alloc(r0.N, r0.H, r0.W, 512);
    { ConvArgs c; c.srcs = {o}; c.ks = 1; c.w = &lin_w(a + ".to_out.0"); c.out = y; c.res1 = &r0; c.want_stats = true; b.conv(a + ".to_out", c); }
    b.release(o);
    b.release(r0);
    T4 r1 = resnet(b, p + ".resnets.1", {y}, 512, 1e-6f, false);
    b.release(y);
    return r1;
  }

  // encode_rgb: genpercept_pipeline.py:488-505
  T4 vae_encoder(Builder& b, const T4& rgb32) {
    const std::string e = "vae.encoder";
    T4 x = b.alloc(rgb32.N, rgb32.H, rgb32.W, 128);
    {   // conv_in over the K-packed input (preprocess_rgb_im2col): a 1x1 GEMM with K = 27
      if (!packed.count(e + ".conv_in#im2col")) {
        const HostT& w = T(e + ".conv_in.weight");
        GP_REQUIRE(w.shape.size() == 4 && w.shape[0] == 128 && w.shape[1] == 3 && w.shape[2] == 3, e + ".conv_in: unexpected shape");
        std::vector<float> m((size_t)128 * 32, 0.f);
        for (int co = 0; co < 128; ++co)
          for (int c = 0; c < 3; ++c)
            for (int r = 0; r < 3; ++r)
              for (int q = 0; q < 3; ++q)
                m[(size_t)co * 32 + im2col_tap_slot(r, q) * 3 + c] = w.d[(((size_t)co * 3 + c) * 3 + r) * 3 + q];
        mat_w(e + ".conv_in#im2col", 128, 32, m.data(), T(e + ".conv_in.bias").d);
      }
      ConvArgs c;
      c.srcs = {rgb32};
      c.ks = 1;
      c.w = &packed.at(e + ".conv_in#im2col");
      c.out = x;
      c.want_stats = true;
      b.conv(e + ".conv_in", c);
    }
    const int ch[5] = {128, 128, 256, 512, 512};
    for (int i = 0; i < 4; ++i) {
      for (int j = 0; j < 2; ++j) {
        T4 y = resnet(b, e + ".down_blocks." + std::to_string(i) + ".resnets." + std::to_string(j), {x}, ch[i + 1], 1e-6f, false);
        b.release(x);
        x = y;
      }
      if (i < 3) {
        const std::string k = e + ".down_blocks." + std::to_string(i) + ".downsamplers.0.conv";
        T4 y = b.alloc(x.N, (x.H + 1 - 3) / 2 + 1, (x.W + 1 - 3) / 2 + 1, x.C);
        ConvArgs c; c.srcs = {x}; c.mode = 2; c.w = &conv_w(k, {x.C}); c.out = y; c.want_stats = true;
        b.conv(k, c);
        b.release(x);
        x = y;
      }
    }
    x = vae_mid(b, e + ".mid_block", x);
    // conv_out (512->8) o quant_conv (8->8), mean channels, * 0.18215  ->  one 3x3 conv 512->4 (App. C.2)
    if (!packed.count("vae.encoder.tail")) {
      const HostT &w = T(e + ".conv_out.weight"), &bb = T(e + ".conv_out.bias"), &q = T("vae.quant_conv.weight"), &qb = T("vae.quant_conv.bias");
      folded["vae.encoder.tail"].assign((size_t)8 * 512 * 9, 0.f);
      std::vector<float>& f = folded["vae.encoder.tail"];
      std::vector<float> bias(8, 0.f);
      for (int o = 0; o < 4; ++o) {
        double bs = qb.d[o];
        for (int m = 0; m < 8; ++m) {
          const float qm = q.d[o * 8 + m];
          bs += (double)qm * bb.d[m];
          for (int i = 0; i < 512 * 9; ++i) f[(size_t)o * 512 * 9 + i] += kLatentScale * qm * w.d[(size_t)m * 512 * 9 + i];
        }
        bias[o] = (float)(kLatentScale * bs);
      }
      std::vector<SegSpec> segs;
      for (int r = 0; r < 9; ++r) { SegSpec sg; sg.C = 512; sg.terms.push_back(Term{f.data() + r, 512 * 9, 9, 1.f}); segs.push_back(sg); }
      packed.emplace("vae.encoder.tail", pack({segs}, 8, bias));
    }
    T4 lat = b.alloc(x.N, x.H, x.W, 8);
    {
      ConvArgs c; c.srcs = {x}; c.w = &packed.at("vae.encoder.tail"); c.out = lat;
      c.gn = &norm_w(e + ".conv_norm_out"); c.gn_name = e + ".conv_norm_out"; c.gn_eps = 1e-6f;
      b.conv("vae.encoder.tail", c);
    }
    b.release(x);
    return lat;
  }

  // UNet2DConditionModel.forward (custom_unet.py); returns z (NHWC8) or, for the DPT readout, the 4 taps
  void unet(Builder& b, const T4& lat8, bool want_feats, T4* z_out, T4 feats[4]) {
    compute_temb();
    const std::string u = "unet";
    T4 x = b.alloc(lat8.N, lat8.H, lat8.W, 320);
    // conv_in takes 4 channels (GenPercept, rgb_blending) or 8 = cat([rgb_latent, pred_latent]) (run.py:59-78, --archs marigold)
    if (unet_in_ch == 0) {
      const HostT& wci = T(u + ".conv_in.weight");
      GP_REQUIRE(wci.shape.size() == 4 && (wci.shape[1] == 4 || wci.shape[1] == 8), "unet.conv_in must take 4 or 8 channels");
      unet_in_ch = (int)wci.shape[1];
      GP_REQUIRE(multistep || unet_in_ch == 4, "an 8-channel conv_in belongs to the multi-step arch (gp_config.arch = 1)");
    }
    small_cin_conv(b, u + ".conv_in", lat8, unet_in_ch, x);
    std::vector<T4> skips = {x};
    for (int i = 0; i < 4; ++i) {
      const int cout = kUnetOut[i];
      for (int j = 0; j < 2; ++j) {
        const std::string rp = u + ".down_blocks." + std::to_string(i) + ".resnets." + std::to_string(j);
        T4 y = resnet(b, rp, {x}, cout, 1e-5f, true);
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
        T4 y = b.alloc(x.N, (x.H + 2 - 3) / 2 + 1, (x.W + 2 - 3) / 2 + 1, x.C);
        ConvArgs c; c.srcs = {x}; c.mode = 1; c.w = &conv_w(k, {x.C}); c.out = y; c.want_stats = true;
        b.conv(k, c);
        x = y;
        skips.push_back(x);
      }
    }
    // mid block; x (the last skip) stays alive for the up path
    T4 m0 = resnet(b, u + ".mid_block.resnets.0", {x}, 1280, 1e-5f, true);
    T4 m1 = transformer(b, u + ".mid_block.attentions.0", m0, 20);
    b.release(m0);
    T4 cur = resnet(b, u + ".mid_block.resnets.1", {m1}, 1280, 1e-5f, true);
    b.release(m1);
    const int up_out[4] = {1280, 1280, 640, 320};
    const bool up_attn[4] = {false, true, true, true};
    const int up_heads[4] = {0, 20, 10, 5};
    for (int i = 0; i < 4; ++i) {
      for (int j = 0; j < 3; ++j) {
        T4 skip = skips.back();
        skips.pop_back();
        const std::string rp = u + ".up_blocks." + std::to_string(i) + ".resnets." + std::to_string(j);
        T4 y = resnet(b, rp, {cur, skip}, up_out[i], 1e-5f, true);
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
        const PackedW& plain = conv_w(k, {cur.C}, "", {}, nullptr, true, "#plain");   // packed at finalize for both paths
        if (nxt.H == 2 * cur.H && nxt.W == 2 * cur.W) {
          T4 y = b.alloc(cur.N, 2 * cur.H, 2 * cur.W, cur.C);
          ConvArgs c; c.srcs = {cur}; c.mode = 3; c.w = &conv_up_w(k); c.out = y; c.want_stats = true;
          b.conv(k, c);
          b.release(cur);
          cur = y;
        } else {
          GP_REQUIRE(nxt.H <= 2 * cur.H && nxt.H >= 2 * cur.H - 1 && nxt.W <= 2 * cur.W && nxt.W >= 2 * cur.W - 1,
                     "unexpected skip size in the UNet up path");
          T4 up = b.alloc(cur.N, nxt.H, nxt.W, cur.C);
          if (!b.measuring()) {
            const void* src = b.ptr(cur);
            void* dst = b.ptr(up);
            const int n = cur.N, h = cur.H, w = cur.W, oh = nxt.H, ow = nxt.W, ch = (int)cur.ps();   // both planes move together
            b.custom(k + ".nearest", 1, (double)cur.bytes() + (double)up.bytes(),
                     [=](cudaStream_t s) { return nearest_resize(src, dst, n, h, w, oh, ow, ch, s); });
          }
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
      if (pq_dev == nullptr) {
        std::vector<float> pqm = T("vae.post_quant_conv.weight").d;
        const std::vector<float>& pqb = T("vae.post_quant_conv.bias").d;
        pqm.insert(pqm.end(), pqb.begin(), pqb.end());
        pq_dev = upload(pqm);
      }
      if (!packed.count("unet.conv_out#plain")) {
        const HostT &w = T(u + ".conv_out.weight"), &bb = T(u + ".conv_out.bias");
        folded["unet.conv_out#plain"].assign((size_t)8 * 320 * 9, 0.f);
        std::vector<float>& f = folded["unet.conv_out#plain"];
        std::copy(w.d.begin(), w.d.begin() + (size_t)4 * 320 * 9, f.begin());
        std::vector<float> bias(8, 0.f);
        for (int o = 0; o < 4; ++o) bias[o] = bb.d[o];
        std::vector<SegSpec> segs;
        for (int r = 0; r < 9; ++r) { SegSpec sg; sg.C = 320; sg.terms.push_back(Term{f.data() + r, 320 * 9, 9, 1.f}); segs.push_back(sg); }
        packed.emplace("unet.conv_out#plain", pack({segs}, 8, bias));
      }
      ConvArgs c; c.srcs = {cur}; c.w = &packed.at("unet.conv_out#plain"); c.out = *z_out;
      c.gn = &norm_w(u + ".conv_norm_out"); c.gn_name = u + ".conv_norm_out"; c.gn_eps = 1e-5f;
      b.conv("unet.conv_out", c);
      b.release(cur);
      return;
    }
    // conv_out, DDIM(beta=1) x0 = -v, /0.18215, post_quant_conv  ->  one 3x3 conv 320->4 (App. C.3)
    if (!packed.count("unet.tail")) {
      if (pq_dev == nullptr) {       // decode_pred of a caller-supplied latent applies post_quant_conv itself (gp_decode)
        std::vector<float> pqm = T("vae.post_quant_conv.weight").d;
        const std::vector<float>& pqb = T("vae.post_quant_conv.bias").d;
        pqm.insert(pqm.end(), pqb.begin(), pqb.end());
        pq_dev = upload(pqm);
      }
      const HostT &w = T(u + ".conv_out.weight"), &bb = T(u + ".conv_out.bias"), &pq = T("vae.post_quant_conv.weight"), &pb = T("vae.post_quant_conv.bias");
      folded["unet.tail"].assign((size_t)8 * 320 * 9, 0.f);
      std::vector<float>& f = folded["unet.tail"];
      std::vector<float> bias(8, 0.f);
      const float k = -1.0f / kLatentScale;
      for (int o = 0; o < 4; ++o) {
        double bs = 0;
        for (int m = 0; m < 4; ++m) {
          const float pm = pq.d[o * 4 + m];
          bs += (double)pm * bb.d[m];
          for (int i = 0; i < 320 * 9; ++i) f[(size_t)o * 320 * 9 + i] += k * pm * w.d[(size_t)m * 320 * 9 + i];
        }
        bias[o] = (float)(k * bs + pb.d[o]);
      }
      std::vector<SegSpec> segs;
      for (int r = 0; r < 9; ++r) { SegSpec sg; sg.C = 320; sg.terms.push_back(Term{f.data() + r, 320 * 9, 9, 1.f}); segs.push_back(sg); }
      packed.emplace("unet.tail", pack({segs}, 8, bias));
    }
    {
      ConvArgs c; c.srcs = {cur}; c.w = &packed.at("unet.tail"); c.out = *z_out;
      c.gn = &norm_w(u + ".conv_norm_out"); c.gn_name = u + ".conv_norm_out"; c.gn_eps = 1e-5f;
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
        T4 y = resnet(b, d + ".up_blocks." + std::to_string(i) + ".resnets." + std::to_string(j), {x}, oc[i], 1e-6f, false);
        b.release(x);
        x = y;
      }
      if (i < 3) {
        const std::string k = d + ".up_blocks." + std::to_string(i) + ".upsamplers.0.conv";
        T4 y = b.alloc(x.N, 2 * x.H, 2 * x.W, x.C);
        ConvArgs c; c.srcs = {x}; c.mode = 3; c.w = &conv_up_w(k); c.out = y; c.want_stats = true;
        b.conv(k, c);
        b.release(x);
        x = y;
      }
    }
    // 3-channel (normal / seg) and channel-mean (depth / matting / dis / disparity) variants
    if (!packed.count("vae.decoder.tail1")) {
      const HostT &w = T(d + ".conv_out.weight"), &bb = T(d + ".conv_out.bias");
      folded["vae.decoder.tail1"].assign((size_t)128 * 9, 0.f);
      std::vector<float>& f = folded["vae.decoder.tail1"];
      for (int m = 0; m < 3; ++m)
        for (int i = 0; i < 128 * 9; ++i) f[i] += w.d[(size_t)m * 128 * 9 + i] / 3.0f;
      std::vector<SegSpec> segs;
      for (int r = 0; r < 9; ++r) { SegSpec sg; sg.C = 128; sg.terms.push_back(Term{f.data() + r, 128 * 9, 9, 1.f}); segs.push_back(sg); }
      packed.emplace("vae.decoder.tail1", pack({segs}, 1, {(bb.d[0] + bb.d[1] + bb.d[2]) / 3.0f}));
      conv_w(d + ".conv_out", {128});
    }
    for (int variant : {1, 3}) {
      b.variant = variant;
      ConvArgs c;
      c.srcs = {x};
      c.gn = &norm_w(d + ".conv_norm_out"); c.gn_name = d + ".conv_norm_out"; c.gn_eps = 1e-6f;
      c.w = variant == 1 ? &packed.at("vae.decoder.tail1") : &packed.at(d + ".conv_out");
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
    { ConvArgs c; c.srcs = {r}; c.w = &conv_w(p + ".convolution1", {256}, "", {}, nullptr, false); c.out = c1; c.flags = IG_RELU; b.conv(p + ".convolution1", c); }
    b.release(r);
    T4 out = b.alloc(x.N, x.H, x.W, 256);
    { ConvArgs c; c.srcs = {c1}; c.w = &conv_w(p + ".convolution2", {256}, "", {}, nullptr, false); c.out = out; c.res1 = &x; c.res2 = extra_res; b.conv(p + ".convolution2", c); }
    b.release(c1);
    return out;
  }
  void dpt_head(Builder& b, T4 feats[4], float* out_f32, unsigned int* mm_scratch, int* out_h, int* out_w) {
    // feats (up-block order): [1280@h/4, 1280@h/2, 640@h, 320@h]; reference reverses (:479)
    T4 f0 = feats[3], f1 = feats[2], f2 = feats[1], f3 = feats[0];
    T4 f0u = b.alloc(f0.N, 2 * f0.H, 2 * f0.W, 320);
    { ConvArgs c; c.srcs = {f0}; c.mode = 3; c.w = &conv_up_w("dpt.feature_upsample_0.conv"); c.out = f0u; b.conv("dpt.feature_upsample_0", c); }
    const T4 fin[4] = {f0u, f1, f2, f3};
    T4 nk[4];
    for (int i = 0; i < 4; ++i) {
      nk[i] = b.alloc(fin[i].N, fin[i].H, fin[i].W, 256);
      ConvArgs c; c.srcs = {fin[i]}; c.w = &conv_w("dpt.neck.convs." + std::to_string(i), {fin[i].C}, "", {}, nullptr, false); c.out = nk[i];
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
          if (!b.measuring()) {
            const void* src = b.ptr(f);
            void* dst = b.ptr(fr);
            const int n = f.N, h = f.H, w = f.W, oh = x.H, ow = x.W;
            const bool bf = bf16, spl = split;
            b.custom(lp + ".resize_skip", 1, (double)f.bytes() + (double)fr.bytes(),
                     [=](cudaStream_t st) { return bilinear_resize(src, dst, n, h, w, oh, ow, 256, bf, st, spl); });
          }
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
      { ConvArgs c; c.srcs = {up}; c.ks = 1; c.w = &lin_w(lp + ".projection"); c.out = x; b.conv(lp + ".projection", c); }
      b.release(up);
    }
    T4 p = b.alloc(x.N, x.H, x.W, 256);
    { ConvArgs c; c.srcs = {x}; c.w = &conv_w("dpt.head.projection", {256}); c.out = p; c.flags = IG_RELU; b.conv("dpt.head.projection", c); }
    b.release(x);
    T4 h0 = b.alloc(p.N, p.H, p.W, 128);
    { ConvArgs c; c.srcs = {p}; c.w = &conv_w("dpt.head.head.0", {256}); c.out = h0; b.conv("dpt.head.head.0", c); }
    b.release(p);
    T4 h1 = b.alloc(h0.N, 2 * h0.H, 2 * h0.W, 128);
    b.bilinear("dpt.head.up", h0, h1);
    b.release(h0);
    T4 h2 = b.alloc(h1.N, h1.H, h1.W, 32);
    { ConvArgs c; c.srcs = {h1}; c.w = &conv_w("dpt.head.head.2", {128}); c.out = h2; c.flags = IG_RELU; b.conv("dpt.head.head.2", c); }
    b.release(h1);
    b.direct("dpt.head.head.4", h2, 32, direct_w("dpt.head.head.4", 32), h2, 0, out_f32, 0);
    const int N = h2.N;
    const long long HW = (long long)h2.H * h2.W;
    *out_h = h2.H; *out_w = h2.W;
    b.release(h2);
    float** slot = b.out_slot;
    b.custom("dpt.minmax", 3, 3.0 * N * HW * 4, [=](cudaStream_t s) { return minmax_normalize(slot ? *slot : out_f32, N, HW, mm_scratch, s); });
  }

  std::unordered_map<std::string, std::vector<float>> folded;   // host fp32 folded weights (live until packed)

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
      plan->kept["rgb"] = Kept{rgb8, nullptr, 3};
      plan->kept["rgb_latent"] = Kept{latent, nullptr, 4};
      if (!dpt) plan->kept["z"] = Kept{z, nullptr, 4};
      if (multistep) {
        plan->kept["xin"] = Kept{xin, nullptr, 8};
        plan->kept["sample"] = Kept{sample, nullptr, 4};
        plan->kept["noise_pred"] = Kept{npred, nullptr, 4};
        plan->kept["x0"] = Kept{x0, nullptr, 4};
      }
      if (dpt)
        for (int i = 0; i < 4; ++i) plan->kept["feat" + std::to_string(i)] = Kept{feats[i], nullptr, feats[i].C};
    }
  }
};

// ------------------------------------------------------------------------------------ C-ABI
namespace {

template <class F>
gp_status guarded(gp_engine* e, F f) {
  if (!e) return GP_ERR_INVALID;
  if (e->poisoned) { e->err = "engine poisoned by an earlier CUDA error: " + e->err; return GP_ERR_CUDA; }
  try {
    f();
    return GP_OK;
  } catch (const GpError& ex) {
    e->err = ex.what();
    if (ex.st == GP_ERR_CUDA) e->poisoned = true;
    return ex.st;
  } catch (const std::exception& ex) {
    e->err = ex.what();
    return GP_ERR_INVALID;
  }
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

}  // namespace

extern "C" {

gp_status gp_create(const gp_config* cfg, gp_engine** out) {
  if (!cfg || !out) return GP_ERR_INVALID;
  *out = nullptr;
  if (cfg->dtype != GP_F16 && cfg->dtype != GP_BF16) return GP_ERR_INVALID;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= cfg->device) return GP_ERR_CUDA;
  if (cudaSetDevice(cfg->device) != cudaSuccess) return GP_ERR_CUDA;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, cfg->device) != cudaSuccess || prop.major != 9) return GP_ERR_CUDA;   // sm_90a only
  gp_engine* e = new gp_engine();
  e->cfg = *cfg;
  if (e->cfg.timestep <= 0) e->cfg.timestep = 1;
  e->bf16 = cfg->dtype == GP_BF16;
  e->split = cfg->precision == 1;
  e->multistep = cfg->arch == 1;
  if (cfg->arch != 0 && cfg->arch != 1) { delete e; return GP_ERR_INVALID; }
  if (cfg->precision != 0 && cfg->precision != 1) { delete e; return GP_ERR_INVALID; }
  *out = e;
  return GP_OK;
}

void gp_destroy(gp_engine* e) {
  if (!e) return;
  for (auto& kv : e->plans) {
    for (auto& g : kv.second->graphs) cudaGraphExecDestroy(g.second);
    if (kv.second->arena) cudaFree(kv.second->arena);
  }
  for (void* p : e->dev_allocs) cudaFree(p);
  delete e;
}

const char* gp_last_error(gp_engine* e) { return e ? e->err.c_str() : "null engine"; }

gp_status gp_load_tensor(gp_engine* e, const char* key, const void* host_ptr, int dtype, const int64_t* shape, int ndim) {
  return guarded(e, [&]() {
    GP_REQUIRE(key && host_ptr && shape && ndim >= 1 && ndim <= 4, "gp_load_tensor: bad arguments");
    if (e->finalized) throw GpError(GP_ERR_STATE, "gp_load_tensor after gp_finalize");
    HostT t;
    t.shape.assign(shape, shape + ndim);
    const int64_t n = t.numel();
    t.d.resize((size_t)n);
    if (dtype == GP_F32) std::memcpy(t.d.data(), host_ptr, (size_t)n * 4);
    else if (dtype == GP_F16 || dtype == GP_BF16) {
      const uint16_t* s = reinterpret_cast<const uint16_t*>(host_ptr);
      for (int64_t i = 0; i < n; ++i) t.d[(size_t)i] = host_h2f(s[i], dtype == GP_BF16);
    } else throw GpError(GP_ERR_INVALID, "gp_load_tensor: unsupported dtype");
    e->host[key] = std::move(t);
  });
}

gp_status gp_set_text_embed(gp_engine* e, const float* host_ptr, int n_tokens, int dim) {
  return guarded(e, [&]() {
    GP_REQUIRE(host_ptr && dim == 1024 && n_tokens >= 1, "gp_set_text_embed: expected [n_tokens, 1024]");
    if (e->finalized) throw GpError(GP_ERR_STATE, "gp_set_text_embed after gp_finalize");
    e->text_embed.assign(host_ptr, host_ptr + (size_t)n_tokens * dim);
    e->n_tokens = n_tokens;
  });
}

gp_status gp_finalize(gp_engine* e) {
  return guarded(e, [&]() {
    if (e->finalized) return;
    GP_REQUIRE(e->n_tokens > 0, "gp_finalize: text embedding not set");
    GP_CUDA(cudaSetDevice(e->cfg.device));
    // A measuring pass over a nominal shape touches every weight the topology needs: packs + uploads.
    Builder b(e->bf16, true, nullptr, e->split);
    e->build(b, nullptr, 1, 64, 64);
    e->folded.clear();
    e->host.clear();
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
    if (it != e->plans.end()) { e->cur = it->second.get(); e->cur->last_used = ++e->use_clock; return; }
    // Bounded plan cache (a folder of in-the-wild images yields a new (H, W) per aspect ratio): evict the least
    // recently used plans — graph execs destroyed, arena freed — before building another one.
    static const size_t max_plans = std::getenv("GP_MAX_PLANS") ? (size_t)std::max(1, std::atoi(std::getenv("GP_MAX_PLANS"))) : 4;
    while (e->plans.size() >= max_plans) {
      auto victim = e->plans.begin();
      for (auto jt = e->plans.begin(); jt != e->plans.end(); ++jt)
        if (jt->second->last_used < victim->second->last_used) victim = jt;
      GP_CUDA(cudaDeviceSynchronize());
      for (auto& g : victim->second->graphs) cudaGraphExecDestroy(g.second);
      if (victim->second->arena) cudaFree(victim->second->arena);
      if (e->cur == victim->second.get()) e->cur = nullptr;
      e->plans.erase(victim);
    }
    Builder m(e->bf16, true, nullptr, e->split);
    e->build(m, nullptr, B, H, W);
    std::unique_ptr<Plan> p(new Plan());
    p->B = B; p->H = H; p->W = W;
    p->arena_bytes = m.arena_bytes();
    const cudaError_t ae = cudaMalloc(reinterpret_cast<void**>(&p->arena), p->arena_bytes);
    if (ae == cudaErrorMemoryAllocation) {
      // Not a sticky error: clear it and report the shape as too large, so the engine stays usable for smaller inputs.
      cudaGetLastError();
      p->arena = nullptr;
      throw GpError(GP_ERR_INVALID, "gp_plan: batch " + std::to_string(B) + " at " + std::to_string(H) + "x" +
                                        std::to_string(W) + " needs an activation arena of " +
                                        std::to_string(p->arena_bytes) + " bytes, more than the device can allocate");
    }
    GP_CUDA(ae);
    GP_CUDA(cudaMemset(p->arena, 0, p->arena_bytes));
    Builder b(e->bf16, false, p->arena, e->split);
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

gp_status gp_tile_shape(int cout, int cin, int ks, int images, int h, int w, int tokens_mode, int num_sms, int* bn, int* mt) {
  if (!bn || !mt || cout < 1 || cin < 1 || ks < 1 || images < 1 || h < 1 || w < 1 || num_sms < 1) return GP_ERR_INVALID;
  gp::tile_shape_for(cout, (double)cin * ks * ks, tokens_mode != 0, images, w, h, num_sms, bn, mt);
  return GP_OK;
}

static void set_timestep_now(gp_engine* e, int timestep);

gp_status gp_set_timestep(gp_engine* e, int timestep) {
  return guarded(e, [&]() { set_timestep_now(e, timestep); });
}

static void set_timestep_now(gp_engine* e, int timestep) {
  {
    if (!e->finalized) throw GpError(GP_ERR_STATE, "gp_set_timestep before gp_finalize");
    GP_REQUIRE(timestep >= 0 && timestep <= 1000, "gp_set_timestep: timestep must be in [0, 1000]");
    if (timestep == e->cur_timestep) return;
    GP_CUDA(cudaSetDevice(e->cfg.device));
    auto it = e->temb_cache.find(timestep);
    if (it == e->temb_cache.end()) {
      const std::vector<float> emb = e->temb_for(timestep);
      std::vector<std::vector<float>> biases(e->temb_layers.size());
      parallel_for((int)e->temb_layers.size(), [&](int i) {
        const auto& tl = e->temb_layers[(size_t)i];
        std::vector<float> b = gp_engine::temb_proj_of(tl.w, tl.b, emb);
        for (int o = 0; o < tl.cout; ++o) b[(size_t)o] += tl.conv_bias[(size_t)o];
        biases[(size_t)i] = std::move(b);
      });
      it = e->temb_cache.emplace(timestep, std::move(biases)).first;
    }
    GP_CUDA(cudaDeviceSynchronize());          // nothing in flight may still read the old biases
    for (size_t i = 0; i < e->temb_layers.size(); ++i)
      GP_CUDA(cudaMemcpy(e->temb_layers[i].dev_bias, it->second[i].data(), (size_t)e->temb_layers[i].cout * 4, cudaMemcpyHostToDevice));
    e->cur_timestep = timestep;
  }
}

gp_status gp_infer(gp_engine* e, const void* rgb, int rgb_dtype, int rgb_on_host, float* out, int out_on_host,
                   int out_channels, void* stream) {
  return guarded(e, [&]() {
    Plan* p = e->cur;
    if (!p) throw GpError(GP_ERR_NO_PLAN, "gp_infer: no plan (call gp_plan)");
    if (e->multistep) throw GpError(GP_ERR_STATE, "gp_infer: this engine runs the multi-step arch (gp_infer_steps)");
    const bool dpt = e->cfg.readout == GP_READOUT_DPT;
    if (dpt) out_channels = 1;
    GP_REQUIRE(rgb && out && (out_channels == 1 || out_channels == 3), "gp_infer: bad arguments");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    GP_CUDA(cudaSetDevice(e->cfg.device));
    p->last_used = ++e->use_clock;
    const size_t npix = (size_t)p->B * p->H * p->W;
    const size_t npix_out = (size_t)p->B * p->outH * p->outW;
    int kind = 0;
    size_t esz = 1;
    if (rgb_dtype == GP_U8) { kind = 0; esz = 1; }
    else if (rgb_dtype == GP_F16) { kind = 1; esz = 2; }
    else if (rgb_dtype == GP_F32) { kind = 2; esz = 4; }
    else throw GpError(GP_ERR_INVALID, "gp_infer: rgb dtype must be u8, f16 or f32");
    // a device input is read where it lies; only host inputs go through the plan's staging buffer
    const void* src = rgb;
    if (rgb_on_host) {
      GP_CUDA(cudaMemcpyAsync(p->in_staging, rgb, npix * 3 * esz, cudaMemcpyHostToDevice, s));
      src = p->in_staging;
    }
    GP_CUDA(preprocess_rgb_im2col(src, kind, p->arena + p->kept["rgb"].t.off, p->B, p->H, p->W, e->bf16, s, e->split));
    // 2 = auto: replay a graph where the launch stream is the bottleneck — small plans
    const bool use_graph = e->cfg.use_cuda_graph == 1 ||
                           (e->cfg.use_cuda_graph == 2 && (long long)p->B * p->H * p->W <= 2LL * 768 * 768);
    // eager launches write the result straight into a device `out`; a captured graph has the plan's own buffer baked in
    const bool graph_now = use_graph && p->eager_runs > 0;
    p->out_dst = (graph_now || out_on_host) ? p->out_f32 : out;
    if (graph_now) {
      auto it = p->graphs.find(out_channels);
      if (it == p->graphs.end()) {
        cudaStream_t cs;
        GP_CUDA(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
        cudaGraph_t g;
        GP_CUDA(cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal));
        cudaError_t re = run_ops(p, GP_STAGE_VAE_ENCODE, GP_STAGE_READOUT, out_channels, cs);
        cudaError_t ce = cudaStreamEndCapture(cs, &g);
        cudaStreamDestroy(cs);
        GP_CUDA(re);
        GP_CUDA(ce);
        cudaGraphExec_t ge;
        GP_CUDA(cudaGraphInstantiate(&ge, g, 0));
        cudaGraphDestroy(g);
        it = p->graphs.emplace(out_channels, ge).first;
      }
      GP_CUDA(cudaGraphLaunch(it->second, s));
    } else {
      GP_CUDA(run_ops(p, GP_STAGE_VAE_ENCODE, GP_STAGE_READOUT, out_channels, s));
      p->eager_runs++;
    }
    if (p->out_dst != out)
      GP_CUDA(cudaMemcpyAsync(out, p->out_f32, npix_out * out_channels * 4, out_on_host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, s));
    p->out_dst = p->out_f32;
    if (rgb_on_host || out_on_host) GP_CUDA(cudaStreamSynchronize(s));
  });
}

gp_status gp_encode(gp_engine* e, const void* rgb, int rgb_dtype, int rgb_on_host, float* latent_dev, void* stream) {
  return guarded(e, [&]() {
    Plan* p = e->cur;
    if (!p) throw GpError(GP_ERR_NO_PLAN, "gp_encode: no plan (call gp_plan)");
    GP_REQUIRE(rgb && latent_dev, "gp_encode: bad arguments");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    GP_CUDA(cudaSetDevice(e->cfg.device));
    int kind = 0;
    size_t esz = 1;
    if (rgb_dtype == GP_U8) { kind = 0; esz = 1; }
    else if (rgb_dtype == GP_F16) { kind = 1; esz = 2; }
    else if (rgb_dtype == GP_F32) { kind = 2; esz = 4; }
    else throw GpError(GP_ERR_INVALID, "gp_encode: rgb dtype must be u8, f16 or f32");
    const void* src = rgb;
    if (rgb_on_host) {
      GP_CUDA(cudaMemcpyAsync(p->in_staging, rgb, (size_t)p->B * p->H * p->W * 3 * esz, cudaMemcpyHostToDevice, s));
      src = p->in_staging;
    }
    GP_CUDA(preprocess_rgb_im2col(src, kind, p->arena + p->kept["rgb"].t.off, p->B, p->H, p->W, e->bf16, s, e->split));
    GP_CUDA(run_ops(p, GP_STAGE_VAE_ENCODE, GP_STAGE_VAE_ENCODE, 1, s));
    const T4& l = p->kept["rgb_latent"].t;
    GP_CUDA(nhwc8_to_nchw_f32(p->arena + l.off, latent_dev, l.N, l.H, l.W, 4, e->bf16, s, e->split));
    if (rgb_on_host) GP_CUDA(cudaStreamSynchronize(s));
  });
}

gp_status gp_decode(gp_engine* e, const float* latent_dev, int apply_post_quant, float* out_dev, int out_channels, void* stream) {
  return guarded(e, [&]() {
    Plan* p = e->cur;
    if (!p) throw GpError(GP_ERR_NO_PLAN, "gp_decode: no plan (call gp_plan)");
    if (e->cfg.readout == GP_READOUT_DPT) throw GpError(GP_ERR_STATE, "gp_decode: the DPT readout has no latent decoder");
    GP_REQUIRE(latent_dev && out_dev && (out_channels == 1 || out_channels == 3), "gp_decode: bad arguments");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    GP_CUDA(cudaSetDevice(e->cfg.device));
    const T4& z = p->kept["z"].t;
    GP_CUDA(nchw4_affine_to_nhwc8(latent_dev, p->arena + z.off, z.N, z.H, z.W, 1.0f / kLatentScale,
                                  apply_post_quant ? e->pq_dev : nullptr, apply_post_quant ? e->pq_dev + 16 : nullptr, e->bf16, s,
                                  e->split));
    p->out_dst = out_dev;
    GP_CUDA(run_ops(p, GP_STAGE_READOUT, GP_STAGE_READOUT, out_channels, s));
    p->out_dst = p->out_f32;
  });
}

gp_status gp_infer_steps(gp_engine* e, const void* rgb, int rgb_dtype, int rgb_on_host, const float* noise, int noise_on_host,
                         const int* timesteps, const float* coeffs, int n_steps, float* out, int out_on_host, int out_channels,
                         void* stream) {
  return guarded(e, [&]() {
    Plan* p = e->cur;
    if (!p) throw GpError(GP_ERR_NO_PLAN, "gp_infer_steps: no plan (call gp_plan)");
    if (!e->multistep) throw GpError(GP_ERR_STATE, "gp_infer_steps needs gp_config.arch = 1");
    GP_REQUIRE(rgb && out && timesteps && coeffs && n_steps >= 1 && (out_channels == 1 || out_channels == 3), "gp_infer_steps: bad arguments");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    GP_CUDA(cudaSetDevice(e->cfg.device));
    p->last_used = ++e->use_clock;
    int kind = 0;
    size_t esz = 1;
    if (rgb_dtype == GP_U8) { kind = 0; esz = 1; }
    else if (rgb_dtype == GP_F16) { kind = 1; esz = 2; }
    else if (rgb_dtype == GP_F32) { kind = 2; esz = 4; }
    else throw GpError(GP_ERR_INVALID, "gp_infer_steps: rgb dtype must be u8, f16 or f32");
    const void* src = rgb;
    if (rgb_on_host) {
      GP_CUDA(cudaMemcpyAsync(p->in_staging, rgb, (size_t)p->B * p->H * p->W * 3 * esz, cudaMemcpyHostToDevice, s));
      src = p->in_staging;
    }
    GP_CUDA(preprocess_rgb_im2col(src, kind, p->arena + p->kept["rgb"].t.off, p->B, p->H, p->W, e->bf16, s, e->split));
    GP_CUDA(run_ops(p, GP_STAGE_VAE_ENCODE, GP_STAGE_VAE_ENCODE, out_channels, s));      // rgb_latent (:416)
    const T4& lat = p->kept["rgb_latent"].t;
    const long long npx = lat.pixels();
    uint8_t* A = p->arena;
    void* smp = A + p->kept["sample"].t.off;
    if (noise) {              // marigold: pred_latent = randn (:418-425; the caller draws it with its generator)
      const float* nd = noise;
      if (noise_on_host) {    // the plan's result buffer is free until the decoder runs
        GP_CUDA(cudaMemcpyAsync(p->out_f32, noise, (size_t)npx * 4 * sizeof(float), cudaMemcpyHostToDevice, s));
        nd = p->out_f32;
      }
      GP_CUDA(nchw4_affine_to_nhwc8(nd, smp, lat.N, lat.H, lat.W, 1.0f, nullptr, nullptr, e->bf16, s, e->split));
    } else {                  // rgb_blending: pred_latent = rgb_latent (:426-427)
      GP_CUDA(cudaMemcpyAsync(smp, A + lat.off, lat.bytes(), cudaMemcpyDeviceToDevice, s));
    }
    for (int i = 0; i < n_steps; ++i) {                                                  // :443-463
      GP_CUDA(latent_pack(A + lat.off, smp, A + p->kept["xin"].t.off, npx, e->unet_in_ch, e->bf16, s, e->split));
      set_timestep_now(e, timesteps[i]);
      GP_CUDA(run_ops(p, GP_STAGE_UNET, GP_STAGE_UNET, out_channels, s));
      GP_CUDA(ddim_step(A + p->kept["noise_pred"].t.off, smp, A + p->kept["x0"].t.off, npx, coeffs + 4 * i, e->bf16, s, e->split));
    }
    // pred_latent = step_output.pred_original_sample (:465); decode_pred (:507-526); clip + shift in the last kernel
    GP_CUDA(latent_affine(A + p->kept["x0"].t.off, A + p->kept["z"].t.off, npx, 1.0f / kLatentScale, e->pq_dev, e->pq_dev + 16,
                          e->bf16, s, e->split));
    p->out_dst = out_on_host ? p->out_f32 : out;
    GP_CUDA(run_ops(p, GP_STAGE_READOUT, GP_STAGE_READOUT, out_channels, s));
    if (p->out_dst != out)
      GP_CUDA(cudaMemcpyAsync(out, p->out_f32, (size_t)p->B * p->outH * p->outW * out_channels * 4, cudaMemcpyDeviceToHost, s));
    p->out_dst = p->out_f32;
    if (rgb_on_host || out_on_host) GP_CUDA(cudaStreamSynchronize(s));
  });
}

gp_status gp_run_stage(gp_engine* e, int stage, int out_channels, void* stream) {
  return guarded(e, [&]() {
    Plan* p = e->cur;
    if (!p) throw GpError(GP_ERR_NO_PLAN, "gp_run_stage: no plan");
    if (e->cfg.readout == GP_READOUT_DPT) out_channels = 1;
    GP_CUDA(cudaSetDevice(e->cfg.device));
    p->out_dst = p->out_f32;
    GP_CUDA(run_ops(p, stage, stage, out_channels, reinterpret_cast<cudaStream_t>(stream)));
  });
}

gp_status gp_tensor_shape(gp_engine* e, const char* name, int64_t shape[4]) {
  return guarded(e, [&]() {
    Plan* p = e->cur;
    if (!p) throw GpError(GP_ERR_NO_PLAN, "no plan");
    if (std::string(name) == "out") { shape[0] = p->B; shape[1] = 3; shape[2] = p->outH; shape[3] = p->outW; return; }
    auto it = p->kept.find(name);
    GP_REQUIRE(it != p->kept.end(), std::string("unknown tensor ") + name);
    shape[0] = it->second.t.N; shape[1] = it->second.creal; shape[2] = it->second.t.H; shape[3] = it->second.t.W;
  });
}

gp_status gp_read_tensor(gp_engine* e, const char* name, float* host_out, size_t cap) {
  return guarded(e, [&]() {
    Plan* p = e->cur;
    if (!p) throw GpError(GP_ERR_NO_PLAN, "no plan");
    GP_CUDA(cudaDeviceSynchronize());
    if (std::string(name) == "out") {
      const size_t n = (size_t)p->B * 3 * p->outH * p->outW;
      GP_REQUIRE(cap >= n, "gp_read_tensor: buffer too small");
      GP_CUDA(cudaMemcpy(host_out, p->out_f32, n * 4, cudaMemcpyDeviceToHost));
      return;
    }
    auto it = p->kept.find(name);
    GP_REQUIRE(it != p->kept.end(), std::string("unknown tensor ") + name);
    const T4& t = it->second.t;
    const int cr = it->second.creal;
    GP_REQUIRE(cap >= (size_t)t.N * cr * t.H * t.W, "gp_read_tensor: buffer too small");
    const size_t ps = (size_t)t.ps();
    std::vector<uint16_t> h((size_t)t.N * t.H * t.W * ps);
    GP_CUDA(cudaMemcpy(h.data(), p->arena + t.off, h.size() * 2, cudaMemcpyDeviceToHost));
    const size_t HW = (size_t)t.H * t.W;
    for (int n = 0; n < t.N; ++n)
      for (size_t px = 0; px < HW; ++px)
        for (int c = 0; c < cr; ++c) {
          const uint16_t* q = &h[((size_t)n * HW + px) * ps + c];
          host_out[((size_t)n * cr + c) * HW + px] = host_h2f(q[0], e->bf16) + (t.planes == 2 ? host_h2f(q[t.C], e->bf16) : 0.f);
        }
  });
}

gp_status gp_write_tensor(gp_engine* e, const char* name, const float* host_in, size_t elems) {
  return guarded(e, [&]() {
    Plan* p = e->cur;
    if (!p) throw GpError(GP_ERR_NO_PLAN, "no plan");
    auto it = p->kept.find(name);
    GP_REQUIRE(it != p->kept.end(), std::string("unknown tensor ") + name);
    const T4& t = it->second.t;
    const int cr = it->second.creal;
    GP_REQUIRE(elems == (size_t)t.N * cr * t.H * t.W, "gp_write_tensor: size mismatch");
    const size_t ps = (size_t)t.ps();
    std::vector<uint16_t> h((size_t)t.N * t.H * t.W * ps, 0);
    const size_t HW = (size_t)t.H * t.W;
    for (int n = 0; n < t.N; ++n)
      for (size_t px = 0; px < HW; ++px)
        for (int c = 0; c < cr; ++c) {
          const float v = host_in[((size_t)n * cr + c) * HW + px];
          uint16_t* q = &h[((size_t)n * HW + px) * ps + c];
          q[0] = host_f2h(v, e->bf16);
          if (t.planes == 2) q[t.C] = host_f2h(v - host_h2f(q[0], e->bf16), e->bf16);
        }
    GP_CUDA(cudaDeviceSynchronize());
    GP_CUDA(cudaMemcpy(p->arena + t.off, h.data(), h.size() * 2, cudaMemcpyHostToDevice));
  });
}

gp_status gp_plan_info(gp_engine* e, int64_t* n_ops, int64_t* n_launches, int64_t* arena_bytes, int64_t* weight_bytes,
                       double* igemm_flops) {
  return guarded(e, [&]() {
    Plan* p = e->cur;
    if (!p) throw GpError(GP_ERR_NO_PLAN, "no plan");
    if (n_ops) *n_ops = (int64_t)p->ops.size();
    if (n_launches) *n_launches = p->launches + 1;   // + preprocess
    if (arena_bytes) *arena_bytes = (int64_t)p->arena_bytes;
    if (weight_bytes) *weight_bytes = (int64_t)e->weight_bytes;
    if (igemm_flops) *igemm_flops = p->igemm_flops;
  });
}

gp_status gp_profile_ops(gp_engine* e, int out_channels, void* stream) {
  return guarded(e, [&]() {
    Plan* p = e->cur;
    if (!p) throw GpError(GP_ERR_NO_PLAN, "no plan");
    if (e->cfg.readout == GP_READOUT_DPT) out_channels = 1;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    cudaEvent_t a, b;
    GP_CUDA(cudaEventCreate(&a));
    GP_CUDA(cudaEventCreate(&b));
    p->out_dst = p->out_f32;
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
    Plan* p = e->cur;
    if (!p) throw GpError(GP_ERR_NO_PLAN, "no plan");
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


// ------------------------------------------------------------------------------------ per-kernel entry points
namespace {

struct TempEngine {
  gp_engine e;
  explicit TempEngine(int dtype) { e.bf16 = dtype == GP_BF16; e.cfg.timestep = 1; }
  ~TempEngine() { for (void* p : e.dev_allocs) cudaFree(p); }
};

template <class F>
gp_status guarded_free(F f) {
  try {
    f();
    return GP_OK;
  } catch (const GpError& ex) {
    fprintf(stderr, "[genpercept_b200] %s\n", ex.what());
    return ex.st;
  } catch (const std::exception& ex) {
    fprintf(stderr, "[genpercept_b200] %s\n", ex.what());
    return GP_ERR_INVALID;
  }
}

void run_all(Builder& b, cudaStream_t s) {
  for (auto& op : b.ops) GP_CUDA(op.run(s));
}

void out_dims(int mode, int H, int W, int* Ho, int* Wo) {
  *Ho = H; *Wo = W;
  if (mode == 1) { *Ho = (H + 2 - 3) / 2 + 1; *Wo = (W + 2 - 3) / 2 + 1; }
  if (mode == 2) { *Ho = (H + 1 - 3) / 2 + 1; *Wo = (W + 1 - 3) / 2 + 1; }
  if (mode == 3) { *Ho = 2 * H; *Wo = 2 * W; }
}

}  // namespace

extern "C" {

gp_status gp_conv2d(int dtype, const void* x, int N, int H, int W, int Cin, const float* w_host, const float* bias_host,
                    int Cout, int ks, int mode, const void* residual, int relu, void* y, int use_direct, void* stream) {
  return guarded_free([&]() {
    GP_REQUIRE(x && w_host && y && (ks == 1 || ks == 3) && mode >= 0 && mode <= 3, "gp_conv2d: bad arguments");
    GP_REQUIRE(dtype == GP_F16 || dtype == GP_BF16, "gp_conv2d: dtype must be f16/bf16");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    TempEngine te(dtype);
    HostT w;
    w.shape = {Cout, Cin, ks, ks};
    w.d.assign(w_host, w_host + (size_t)Cout * Cin * ks * ks);
    te.e.host["t.weight"] = std::move(w);
    if (bias_host) {
      HostT b;
      b.shape = {Cout};
      b.d.assign(bias_host, bias_host + Cout);
      te.e.host["t.bias"] = std::move(b);
    }
    int Ho, Wo;
    out_dims(mode, H, W, &Ho, &Wo);
    Builder b(te.e.bf16, false, nullptr);
    T4 xin = b.external(x, N, H, W, Cin);
    T4 yout = b.external(y, N, Ho, Wo, Cout);
    T4 res;
    if (residual) res = b.external(residual, N, Ho, Wo, Cout);
    if (use_direct) {
      const DirectW& dw = te.e.direct_w("t", Cin);
      DirectConvParams p;
      std::memset(&p, 0, sizeof(p));
      p.in = x; p.N = N; p.H = H; p.W = W; p.Cin = Cin; p.in_cstride = Cin;
      p.w = dw.w; p.bias = dw.bias; p.res = residual;
      p.out = y; p.Ho = Ho; p.Wo = Wo; p.Cout = Cout; p.out_cstride = Cout;
      p.ks = ks;
      p.stride = (mode == 1 || mode == 2) ? 2 : 1;
      p.pad = (mode == 2) ? 0 : ks / 2;
      p.flags = (relu ? DC_RELU : 0) | (mode == 3 ? DC_UP2X : 0);
      GP_CUDA(direct_conv(p, te.e.bf16, s));
    } else {
      ConvArgs c;
      c.srcs = {xin};
      c.ks = ks;
      c.mode = mode;
      if (mode == 3) {
        if (!bias_host) { HostT bz; bz.shape = {Cout}; bz.d.assign(Cout, 0.f); te.e.host["t.bias"] = std::move(bz); }
        c.w = &te.e.conv_up_w("t");
      } else {
        c.w = &te.e.conv_w("t", {Cin});
      }
      c.out = yout;
      if (residual) c.res1 = &res;
      c.flags = relu ? IG_RELU : 0;
      b.conv("gp_conv2d", c);
      run_all(b, s);
    }
    GP_CUDA(cudaStreamSynchronize(s));
  });
}

gp_status gp_groupnorm(int dtype, const void* x, int N, int H, int W, int C, int groups, const float* gamma_host,
                       const float* beta_host, float eps, int silu, void* y, void* stream) {
  return guarded_free([&]() {
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    TempEngine te(dtype);
    NormW nw;
    nw.C = C;
    nw.gamma = te.e.upload(std::vector<float>(gamma_host, gamma_host + C));
    nw.beta = te.e.upload(std::vector<float>(beta_host, beta_host + C));
    float* ss = te.e.upload(std::vector<float>((size_t)N * C * 2, 0.f));
    void* arena = nullptr;
    {
      Builder m(te.e.bf16, true, nullptr);
      m.gn("gp_groupnorm", {m.external(x, N, H, W, C)}, nw, groups, eps, silu != 0, m.external(y, N, H, W, C));
      GP_CUDA(cudaMalloc(&arena, m.arena_bytes() + 1024));
      te.e.dev_allocs.push_back(arena);
    }
    // external tensors are addressed relative to the scratch arena's base
    Builder b(te.e.bf16, false, reinterpret_cast<uint8_t*>(arena));
    b.gn_ss = ss;
    b.gn("gp_groupnorm", {b.external(x, N, H, W, C)}, nw, groups, eps, silu != 0, b.external(y, N, H, W, C));
    run_all(b, s);
    GP_CUDA(cudaStreamSynchronize(s));
  });
}

gp_status gp_gn_conv3x3(int dtype, const void* x, int N, int H, int W, int Cin, int groups, const float* gamma_host,
                        const float* beta_host, float eps, int silu, const float* w_host, const float* bias_host, int Cout,
                        const void* sc_x, int Csc, const float* sc_w_host, const float* sc_b_host, const void* residual,
                        void* y, int out_f32, void* stream) {
  return guarded_free([&]() {
    GP_REQUIRE(x && w_host && y && gamma_host && beta_host, "gp_gn_conv3x3: bad arguments");
    GP_REQUIRE(dtype == GP_F16 || dtype == GP_BF16, "gp_gn_conv3x3: dtype must be f16/bf16");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    TempEngine te(dtype);
    auto put = [&](const char* k, std::vector<int64_t> shape, const float* d) {
      HostT t;
      t.shape = shape;
      t.d.assign(d, d + t.numel());
      te.e.host[k] = std::move(t);
    };
    put("t.weight", {Cout, Cin, 3, 3}, w_host);
    std::vector<float> zb(Cout, 0.f);
    put("t.bias", {Cout}, bias_host ? bias_host : zb.data());
    if (sc_x) {
      GP_REQUIRE(sc_w_host != nullptr, "gp_gn_conv3x3: shortcut weights missing");
      put("s.weight", {Cout, Csc, 1, 1}, sc_w_host);
      put("s.bias", {Cout}, sc_b_host ? sc_b_host : zb.data());
    }
    NormW nw;
    nw.C = Cin;
    nw.gamma = te.e.upload(std::vector<float>(gamma_host, gamma_host + Cin));
    nw.beta = te.e.upload(std::vector<float>(beta_host, beta_host + Cin));
    float* ss = te.e.upload(std::vector<float>((size_t)N * Cin * 2, 0.f));
    const PackedW& pw = sc_x ? te.e.conv_w("t", {Cin}, "s", {Csc}) : te.e.conv_w("t", {Cin});
    auto emit = [&](Builder& b) {
      ConvArgs c;
      c.srcs = {b.external(x, N, H, W, Cin)};
      c.gn = &nw; c.gn_name = "gn"; c.gn_groups = groups; c.gn_eps = eps; c.gn_silu = silu != 0;
      c.w = &pw;
      T4 res;
      if (sc_x) c.sc = {b.external(sc_x, N, H, W, Csc)};
      if (residual) { res = b.external(residual, N, H, W, Cout); c.res1 = &res; }
      if (out_f32) { c.out_f32 = reinterpret_cast<float*>(y); c.cout_valid = Cout; c.out = b.external(x, N, H, W, Cin); }
      else c.out = b.external(y, N, H, W, Cout);
      b.conv("gp_gn_conv3x3", c);
    };
    void* arena = nullptr;
    {
      Builder m(te.e.bf16, true, nullptr);
      emit(m);
      GP_CUDA(cudaMalloc(&arena, m.arena_bytes() + 1024));
      te.e.dev_allocs.push_back(arena);
    }
    Builder b(te.e.bf16, false, reinterpret_cast<uint8_t*>(arena));
    b.gn_ss = ss;
    emit(b);
    run_all(b, s);
    GP_CUDA(cudaStreamSynchronize(s));
  });
}

gp_status gp_layernorm(int dtype, const void* x, int64_t tokens, int C, const float* gamma_host, const float* beta_host,
                       float eps, void* y, void* stream) {
  return guarded_free([&]() {
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    TempEngine te(dtype);
    float* g = te.e.upload(std::vector<float>(gamma_host, gamma_host + C));
    float* bt = te.e.upload(std::vector<float>(beta_host, beta_host + C));
    GP_CUDA(layernorm(x, y, tokens, C, g, bt, eps, te.e.bf16, s));
    GP_CUDA(cudaStreamSynchronize(s));
  });
}

gp_status gp_attention(int dtype, const void* q, const void* k, const void* v, int B, int T, int heads, int d, float scale,
                       void* o, void* stream) {
  return guarded_free([&]() {
    // q is pre-scaled by the caller-visible `scale` through an identity-weight GEMM so that the same
    // igemm paths the engine uses (QK^T, softmax, V^T, PV) are exercised.
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    TempEngine te(dtype);
    const int C = heads * d;
    std::vector<float> eye((size_t)C * C, 0.f), eyes((size_t)C * C, 0.f);
    for (int i = 0; i < C; ++i) { eye[(size_t)i * C + i] = 1.f; eyes[(size_t)i * C + i] = scale; }
    const PackedW& wv = te.e.mat_w("eye", C, C, eye.data(), {});
    const PackedW& wq = te.e.mat_w("eyes", C, C, eyes.data(), {});
    const int Tp = (T + 7) / 8 * 8;
    void *qs = nullptr, *vT = nullptr, *arena = nullptr;
    GP_CUDA(cudaMalloc(&qs, (size_t)B * T * C * 2));
    GP_CUDA(cudaMalloc(&vT, (size_t)B * C * Tp * 2));
    te.e.dev_allocs.push_back(qs);
    te.e.dev_allocs.push_back(vT);
    // measuring pass for the scratch (S matrix) size
    {
      Builder m(te.e.bf16, true, nullptr);
      m.attention_qkv("a", nullptr, nullptr, C, nullptr, B, T, heads, d, nullptr, T4{});
      GP_CUDA(cudaMalloc(&arena, m.arena_bytes()));
      te.e.dev_allocs.push_back(arena);
    }
    Builder b(te.e.bf16, false, reinterpret_cast<uint8_t*>(arena));
    T4 qin = b.external(q, B, 1, T, C), qsc = b.external(qs, B, 1, T, C), vin = b.external(v, B, 1, T, C);
    { ConvArgs c; c.srcs = {qin}; c.ks = 1; c.w = &wq; c.out = qsc; b.conv("scale_q", c); }
    {  // V^T via the engine's swapped-operand GEMM with identity weights
      IgemmParams p;
      std::memset(&p, 0, sizeof(p));
      p.flags = te.e.bf16 ? IG_BF16 : 0;
      p.gridW = C; p.gridH = 1; p.TW = 128; p.TH = 1; p.tw_shift = 7;
      p.Z1 = B; p.Z0 = 1; p.b_z_z1 = 1;
      p.nseg[0] = 1;
      p.seg[0][0] = IgemmSeg{0, 0, 0, (uint16_t)(wv.ktot / 64)};
      p.out = vT; p.outW = C; p.outH = 1; p.out_pix_stride = Tp; p.out_z1 = (long long)C * Tp;
      p.out_sy = p.out_sx = 1;
      p.Cout = T;
      p.BN = choose_bn(T, 0);
      GP_CUDA(make_tmap_a(&p.tmA[0], wv.w, wv.ktot, C, 1, 1, wv.ktot, (long long)C * wv.ktot, (long long)C * wv.ktot, 128, 1, te.e.bf16));
      for (int i = 1; i < 4; ++i) p.tmA[i] = p.tmA[0];
      GP_CUDA(make_tmap_b(&p.tmB, b.ptr(vin), C, T, B, C, (long long)T * C, p.BN, te.e.bf16));
      const char* err = igemm_finalize(&p);
      GP_REQUIRE(err == nullptr, std::string("vT: ") + (err ? err : ""));
      b.custom("vT", 1, 0, [p](cudaStream_t st) { return igemm_launch(p, st); });
    }
    b.attention_qkv("attn", qs, k, C, vT, B, T, heads, d, nullptr, b.external(o, B, 1, T, C));
    run_all(b, s);
    GP_CUDA(cudaStreamSynchronize(s));
  });
}

gp_status gp_ensemble_reduce(const float* pred_dev, int B, int H, int W, const float* scale_host, const float* shift_host,
                             int median, int normalise, float* out_dev, void* stream) {
  return guarded_free([&]() {
    GP_REQUIRE(pred_dev && out_dev && scale_host && shift_host && B >= 1 && B <= 32, "gp_ensemble_reduce: bad arguments (B <= 32)");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    float* ss = nullptr;
    GP_CUDA(cudaMalloc(reinterpret_cast<void**>(&ss), (size_t)(2 * B + 2) * sizeof(float)));
    cudaError_t err = cudaMemcpyAsync(ss, scale_host, (size_t)B * 4, cudaMemcpyHostToDevice, s);
    if (err == cudaSuccess) err = cudaMemcpyAsync(ss + B, shift_host, (size_t)B * 4, cudaMemcpyHostToDevice, s);
    const long long HW = (long long)H * W;
    if (err == cudaSuccess) err = ensemble_reduce(pred_dev, B, HW, ss, ss + B, median != 0, out_dev, s);
    // (depth - min) / (max - min).clamp(1e-6), or depth / max for scale-only alignment (ensemble.py:193-201)
    if (err == cudaSuccess && normalise)
      err = minmax_normalize(out_dev, 1, HW, reinterpret_cast<unsigned int*>(ss + 2 * B), s, 1e-6f, normalise == 2);
    cudaError_t e2 = cudaStreamSynchronize(s);
    cudaFree(ss);
    GP_CUDA(err);
    GP_CUDA(e2);
  });
}

gp_status gp_bilinear_up2x(int dtype, const void* x, int N, int H, int W, int C, void* y, void* stream) {
  return guarded_free([&]() {
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    GP_CUDA(bilinear_up2x(x, y, N, H, W, C, dtype == GP_BF16, s));
    GP_CUDA(cudaStreamSynchronize(s));
  });
}

gp_status gp_bench_conv(int dtype, int N, int H, int W, int Cin, int Cout, int ks, int mode, int iters, double* usec,
                        double* flops) {
  return guarded_free([&]() {
    TempEngine te(dtype);
    HostT w;
    w.shape = {Cout, Cin, ks, ks};
    w.d.assign((size_t)Cout * Cin * ks * ks, 0.01f);
    te.e.host["t.weight"] = std::move(w);
    HostT bz;
    bz.shape = {Cout};
    bz.d.assign(Cout, 0.f);
    te.e.host["t.bias"] = std::move(bz);
    int Ho, Wo;
    out_dims(mode, H, W, &Ho, &Wo);
    void *x = nullptr, *y = nullptr;
    GP_CUDA(cudaMalloc(&x, (size_t)N * H * W * Cin * 2));
    GP_CUDA(cudaMalloc(&y, (size_t)N * Ho * Wo * Cout * 2));
    te.e.dev_allocs.push_back(x);
    te.e.dev_allocs.push_back(y);
    GP_CUDA(cudaMemset(x, 0, (size_t)N * H * W * Cin * 2));
    Builder b(te.e.bf16, false, nullptr);
    ConvArgs c;
    c.srcs = {b.external(x, N, H, W, Cin)};
    c.ks = ks; c.mode = mode;
    c.w = (mode == 3) ? &te.e.conv_up_w("t") : &te.e.conv_w("t", {Cin});
    c.out = b.external(y, N, Ho, Wo, Cout);
    b.conv("bench", c);
    cudaEvent_t e0, e1;
    GP_CUDA(cudaEventCreate(&e0));
    GP_CUDA(cudaEventCreate(&e1));
    for (int i = 0; i < 3; ++i) run_all(b, 0);
    GP_CUDA(cudaEventRecord(e0, 0));
    for (int i = 0; i < iters; ++i) run_all(b, 0);
    GP_CUDA(cudaEventRecord(e1, 0));
    GP_CUDA(cudaEventSynchronize(e1));
    float ms = 0;
    GP_CUDA(cudaEventElapsedTime(&ms, e0, e1));
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    if (usec) *usec = ms * 1000.0 / iters;
    if (flops) *flops = b.ops[0].flops;
  });
}

gp_status gp_bench_attention(int dtype, int B, int T, int fused, int iters, double* usec, double* flops) {
  return guarded_free([&]() {
    GP_REQUIRE(dtype == GP_F16 || dtype == GP_BF16, "gp_bench_attention: dtype must be f16/bf16");
    GP_REQUIRE(B >= 1 && T >= 1 && iters >= 1, "gp_bench_attention: bad arguments");
    TempEngine te(dtype);
    const int C = 512;
    const int Tp = (T + 7) / 8 * 8;
    // The VAE mid-block's operands: q | k packed at a pixel stride of 2C, V^T [B][C][Tp], out [B][T][C].
    const size_t qk_n = (size_t)B * T * 2 * C, vt_n = (size_t)B * C * Tp, o_n = (size_t)B * T * C;
    void *qk = nullptr, *vT = nullptr, *o = nullptr, *arena = nullptr;
    GP_CUDA(cudaMalloc(&qk, qk_n * 2));
    te.e.dev_allocs.push_back(qk);
    GP_CUDA(cudaMalloc(&vT, vt_n * 2));
    te.e.dev_allocs.push_back(vT);
    GP_CUDA(cudaMalloc(&o, o_n * 2));
    te.e.dev_allocs.push_back(o);
    // Small pseudo-random operands (scores of order one, as in the model) rather than zeros, so the tensor cores switch
    // as they do on real data.
    {
      std::vector<uint16_t> pat((size_t)1 << 20);
      uint32_t x = 12345u;
      for (auto& v : pat) {
        x = x * 1664525u + 1013904223u;
        const float f = ((int)(x >> 9) - (1 << 22)) * (0.3f / (1 << 22));
        v = host_f2h(f, te.e.bf16);
      }
      for (auto [buf, n] : {std::make_pair(qk, qk_n), std::make_pair(vT, vt_n)})
        for (size_t i = 0; i < n; i += pat.size())
          GP_CUDA(cudaMemcpy(reinterpret_cast<uint16_t*>(buf) + i, pat.data(), std::min(pat.size(), n - i) * 2,
                             cudaMemcpyHostToDevice));
    }
    {
      Builder m(te.e.bf16, true, nullptr);
      m.attn512_path = fused ? 1 : 0;
      m.attention_qkv("a", nullptr, nullptr, 2 * C, nullptr, B, T, 1, C, nullptr, T4{});
      if (m.arena_bytes()) {
        GP_CUDA(cudaMalloc(&arena, m.arena_bytes()));
        te.e.dev_allocs.push_back(arena);
      }
    }
    Builder b(te.e.bf16, false, reinterpret_cast<uint8_t*>(arena));
    b.attn512_path = fused ? 1 : 0;
    b.attention_qkv("attn", qk, reinterpret_cast<uint16_t*>(qk) + C, 2 * C, vT, B, T, 1, C, nullptr,
                    b.external(o, B, 1, T, C));
    cudaEvent_t e0, e1;
    GP_CUDA(cudaEventCreate(&e0));
    GP_CUDA(cudaEventCreate(&e1));
    run_all(b, 0);
    GP_CUDA(cudaDeviceSynchronize());
    GP_CUDA(cudaEventRecord(e0, 0));
    for (int i = 0; i < iters; ++i) run_all(b, 0);
    GP_CUDA(cudaEventRecord(e1, 0));
    GP_CUDA(cudaEventSynchronize(e1));
    float ms = 0;
    GP_CUDA(cudaEventElapsedTime(&ms, e0, e1));
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    if (usec) *usec = ms * 1000.0 / iters;
    if (flops) *flops = 4.0 * B * (double)T * T * C;
  });
}

}  // extern "C"
