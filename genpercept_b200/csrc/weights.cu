// The weight store: checkpoint tensors on the host, constant folding + weight packing (SURVEY.md App. C), the device
// uploads, and the re-fold of the timestep-dependent biases.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <cmath>
#include <cstring>
#include <thread>

#include "engine.h"

namespace gp {

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

namespace {

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

// K segments of a [rows][cin][ks][ks] fp32 array, tap-major: per tap, one segment for each source of `srcC` (sum = cin)
std::vector<SegSpec> tap_segs(const float* w, int cin, int ks, const std::vector<int>& srcC) {
  std::vector<SegSpec> segs;
  for (int r = 0; r < ks; ++r)
    for (int s = 0; s < ks; ++s) {
      int c0 = 0;
      for (int c : srcC) {
        SegSpec sg;
        sg.C = c;
        sg.terms.push_back(Term{w + (long long)c0 * ks * ks + r * ks + s, (long long)cin * ks * ks, ks * ks, 1.f});
        segs.push_back(sg);
        c0 += c;
      }
    }
  return segs;
}

std::vector<float> temb_proj_of(const std::vector<float>& w, const std::vector<float>& b, const std::vector<float>& emb) {
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

}  // namespace

WeightStore::~WeightStore() {
  for (void* p : dev_allocs) cudaFree(p);
}

// ------------------------------------------------------------------ host tensor access
const HostT& WeightStore::T(const std::string& k) const {
  auto it = host.find(k);
  if (it == host.end()) throw GpError(GP_ERR_MISSING, "missing checkpoint tensor: " + k);
  return it->second;
}

void WeightStore::put(const std::string& key, std::vector<int64_t> shape, const float* d) {
  HostT t;
  t.shape = std::move(shape);
  t.d.assign(d, d + t.numel());
  host[key] = std::move(t);
}

void* WeightStore::device_alloc(size_t bytes) {
  void* d = nullptr;
  GP_CUDA(cudaMalloc(&d, bytes));
  dev_allocs.push_back(d);
  return d;
}

// ------------------------------------------------------------------ packing
// [nz][rows][ktot] 16-bit K-major; each segment padded to a multiple of 64 channels.
PackedW WeightStore::pack(const std::vector<std::vector<SegSpec>>& classes, int rows, const std::vector<float>& bias) {
  PackedW w;
  w.rows = rows;
  w.nz = (int)classes.size();
  int ktot = 0;
  for (auto& s : classes[0]) ktot += ceil_div(s.C, 64) * 64;
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
        k0 += ceil_div(sg.C, 64) * 64;
      }
    });
  }
  w.w = upload(buf);
  if (!bias.empty()) {
    GP_REQUIRE((int)bias.size() == rows, "bias size mismatch");
    std::vector<float> b = bias;
    b.resize(ceil_div(rows, 32) * 32 + 32, 0.f);   // float4 loads may run into the padding
    w.bias = upload(b);
  }
  return w;
}

// 3x3 (or 1x1) convolution weights, tap-major, sources concatenated; optional fused 1x1 shortcut
const PackedW& WeightStore::conv_w(const std::string& key, const std::vector<int>& srcC, const std::string& sc_key,
                                   const std::vector<int>& scC, const std::vector<float>* extra_bias, bool want_bias,
                                   const std::string& cache_suffix) {
  auto it = packed.find(key + cache_suffix);
  if (it != packed.end()) return it->second;
  const HostT& w = T(key + ".weight");
  GP_REQUIRE(w.shape.size() == 4, key + ": conv weight must be 4-D");
  const int cout = (int)w.shape[0], cin = (int)w.shape[1], ks = (int)w.shape[2];
  int sum = 0;
  for (int c : srcC) sum += c;
  GP_REQUIRE(sum == cin, key + ": source channels != Cin");
  std::vector<SegSpec> segs = tap_segs(w.d.data(), cin, ks, srcC);
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
const PackedW& WeightStore::conv_up_w(const std::string& key) {
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

const PackedW& WeightStore::mat_w(const std::string& cache_key, int rows, int K, const float* m,
                                  const std::vector<float>& bias) {
  auto it = packed.find(cache_key);
  if (it != packed.end()) return it->second;
  SegSpec sg;
  sg.C = K;
  sg.terms.push_back(Term{m, (long long)K, 1, 1.f});
  return packed.emplace(cache_key, pack({{sg}}, rows, bias)).first->second;
}
const PackedW& WeightStore::lin_w(const std::string& key, bool bias) {
  auto it = packed.find(key);
  if (it != packed.end()) return it->second;
  const HostT& w = T(key + ".weight");
  const int rows = (int)w.shape[0], K = (int)(w.numel() / rows);   // also accepts 1x1 conv weights
  return mat_w(key, rows, K, w.d.data(), bias ? T(key + ".bias").d : std::vector<float>());
}
const NormW& WeightStore::norm_w(const std::string& key) {
  auto it = norms.find(key);
  if (it != norms.end()) return it->second;
  NormW n;
  n.C = (int)T(key + ".weight").d.size();
  n.gamma = upload(T(key + ".weight").d);
  n.beta = upload(T(key + ".bias").d);
  return norms.emplace(key, n).first->second;
}
const DirectW& WeightStore::direct_w(const std::string& key, int cin_used, const std::vector<float>* w_override,
                                     const std::vector<float>* b_override, int cout_override) {
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
const XattnW& WeightStore::xattn_w(const std::string& blk /* ...transformer_blocks.0 */, int C, int heads) {
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
WeightStore::XattnGen WeightStore::xattn_general_w(const std::string& blk, int C, int heads) {
  const int n = n_tokens, d = C / heads;
  const int Kp = (heads * n + 63) / 64 * 64;
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
  return XattnGen{&packed.at(blk + ".attn2.A"), &packed.at(blk + ".attn2.B"), Kp};
}

// ------------------------------------------------------------------ folded weights
// ResNet conv1; in the UNet its bias also takes time_emb_proj(silu(emb(t))) (SURVEY.md F8), and the layer is recorded
// so that set_timestep can re-fold the bias for another timestep.
const PackedW& WeightStore::resnet_conv1(const std::string& p, int cin, bool temb_on) {
  auto it = packed.find(p + ".conv1");
  if (it != packed.end()) return it->second;
  if (!temb_on) return conv_w(p + ".conv1", {cin});
  TembLayer tl;
  tl.key = p;
  tl.w = T(p + ".time_emb_proj.weight").d;
  tl.b = T(p + ".time_emb_proj.bias").d;
  tl.conv_bias = T(p + ".conv1.bias").d;
  const std::vector<float> tp = temb_proj_of(tl.w, tl.b, temb);   // time_emb_proj(silu(emb)), SURVEY.md F8
  const PackedW& w = conv_w(p + ".conv1", {cin}, "", {}, &tp);
  tl.dev_bias = w.bias;
  tl.cout = w.rows;
  temb_layers.push_back(std::move(tl));
  return w;
}

// self-attention [to_q * d^-1/2 ; to_k]: one GEMM writes q | k
const PackedW& WeightStore::self_attn_qk(const std::string& blk, int C, int heads) {
  auto it = packed.find(blk + ".attn1.to_qk");
  if (it != packed.end()) return it->second;
  const HostT &wq = T(blk + ".attn1.to_q.weight"), &wk = T(blk + ".attn1.to_k.weight");
  const float scale = 1.0f / std::sqrt((float)(C / heads));
  std::vector<float> m((size_t)2 * C * C);
  for (size_t i = 0; i < (size_t)C * C; ++i) { m[i] = wq.d[i] * scale; m[(size_t)C * C + i] = wk.d[i]; }
  return mat_w(blk + ".attn1.to_qk", 2 * C, C, m.data(), {});
}

// GEGLU fused into the projection's epilogue: weight rows interleaved [16 values | 16 gates] per
// 32-column chunk so one thread holds a value and its gate; the 8C-wide tensor is never written.
const PackedW& WeightStore::geglu_w(const std::string& blk, int C) {
  auto it = packed.find(blk + ".ff.geglu_w");
  if (it != packed.end()) return it->second;
  const HostT &w = T(blk + ".ff.net.0.proj.weight"), &bb = T(blk + ".ff.net.0.proj.bias");
  const int C4 = 4 * C;
  std::vector<float> m((size_t)8 * C * C), bias(8 * C);
  for (int r = 0; r < 8 * C; ++r) {
    const int chunk = r / 32, q = r % 32;
    const int src = q < 16 ? chunk * 16 + q : C4 + chunk * 16 + (q - 16);
    std::memcpy(&m[(size_t)r * C], &w.d[(size_t)src * C], (size_t)C * sizeof(float));
    bias[r] = bb.d[src];
  }
  return mat_w(blk + ".ff.geglu_w", 8 * C, C, m.data(), bias);
}

// VAE mid-block attention [to_q * 512^-1/2 ; to_k] with both biases
const PackedW& WeightStore::vae_attn_qk(const std::string& a) {
  auto it = packed.find(a + ".to_qk");
  if (it != packed.end()) return it->second;
  const HostT &wq = T(a + ".to_q.weight"), &wk = T(a + ".to_k.weight"), &bq = T(a + ".to_q.bias"), &bk = T(a + ".to_k.bias");
  const float scale = 1.0f / std::sqrt(512.0f);
  std::vector<float> m((size_t)1024 * 512), bias(1024);
  for (size_t i = 0; i < (size_t)512 * 512; ++i) { m[i] = wq.d[i] * scale; m[(size_t)512 * 512 + i] = wk.d[i]; }
  for (int i = 0; i < 512; ++i) { bias[i] = bq.d[i] * scale; bias[512 + i] = bk.d[i]; }
  return mat_w(a + ".to_qk", 1024, 512, m.data(), bias);
}

// softmax rows sum to 1 -> the V bias passes through P.V unchanged: the PV epilogue adds it (512 values + 64 of padding)
const float* WeightStore::vae_v_bias(const std::string& a) {
  auto it = v_biases.find(a);
  if (it != v_biases.end()) return it->second;
  std::vector<float> bv = T(a + ".to_v.bias").d;
  bv.resize(512 + 64, 0.f);
  return v_biases.emplace(a, upload(bv)).first->second;
}

// the VAE encoder's conv_in over the K-packed input (preprocess_rgb_im2col): a 1x1 GEMM with K = 27
const PackedW& WeightStore::encoder_conv_in() {
  const std::string e = "vae.encoder";
  auto it = packed.find(e + ".conv_in#im2col");
  if (it != packed.end()) return it->second;
  const HostT& w = T(e + ".conv_in.weight");
  GP_REQUIRE(w.shape.size() == 4 && w.shape[0] == 128 && w.shape[1] == 3 && w.shape[2] == 3, e + ".conv_in: unexpected shape");
  std::vector<float> m((size_t)128 * 32, 0.f);
  for (int co = 0; co < 128; ++co)
    for (int c = 0; c < 3; ++c)
      for (int r = 0; r < 3; ++r)
        for (int q = 0; q < 3; ++q)
          m[(size_t)co * 32 + im2col_tap_slot(r, q) * 3 + c] = w.d[(((size_t)co * 3 + c) * 3 + r) * 3 + q];
  return mat_w(e + ".conv_in#im2col", 128, 32, m.data(), T(e + ".conv_in.bias").d);
}

// conv_out (512->8) o quant_conv (8->8), mean channels, * 0.18215  ->  one 3x3 conv 512->4 (App. C.2)
const PackedW& WeightStore::encoder_tail() {
  const std::string e = "vae.encoder";
  auto it = packed.find("vae.encoder.tail");
  if (it != packed.end()) return it->second;
  const HostT &w = T(e + ".conv_out.weight"), &bb = T(e + ".conv_out.bias"), &q = T("vae.quant_conv.weight"), &qb = T("vae.quant_conv.bias");
  std::vector<float> f((size_t)8 * 512 * 9, 0.f);
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
  return packed.emplace("vae.encoder.tail", pack({tap_segs(f.data(), 512, 3, {512})}, 8, bias)).first->second;
}

// The multi-step archs run a real scheduler step, and a caller-supplied latent is decoded by gp_decode: both apply
// post_quant_conv outside the graph, with these values.
void WeightStore::upload_post_quant() {
  if (pq_dev != nullptr) return;
  std::vector<float> pqm = T("vae.post_quant_conv.weight").d;
  const std::vector<float>& pqb = T("vae.post_quant_conv.bias").d;
  pqm.insert(pqm.end(), pqb.begin(), pqb.end());
  pq_dev = upload(pqm);
}

// the UNet's conv_out as it is (model_output of a real scheduler step), 4 of 8 rows used; uploads post_quant_conv
const PackedW& WeightStore::unet_conv_out_plain() {
  const std::string u = "unet";
  auto it = packed.find("unet.conv_out#plain");
  if (it != packed.end()) return it->second;
  upload_post_quant();
  const HostT &w = T(u + ".conv_out.weight"), &bb = T(u + ".conv_out.bias");
  std::vector<float> f((size_t)8 * 320 * 9, 0.f);
  std::copy(w.d.begin(), w.d.begin() + (size_t)4 * 320 * 9, f.begin());
  std::vector<float> bias(8, 0.f);
  for (int o = 0; o < 4; ++o) bias[o] = bb.d[o];
  return packed.emplace("unet.conv_out#plain", pack({tap_segs(f.data(), 320, 3, {320})}, 8, bias)).first->second;
}

// conv_out, DDIM(beta=1) x0 = -v, /0.18215, post_quant_conv  ->  one 3x3 conv 320->4 (App. C.3); uploads post_quant_conv
const PackedW& WeightStore::unet_tail() {
  const std::string u = "unet";
  auto it = packed.find("unet.tail");
  if (it != packed.end()) return it->second;
  upload_post_quant();
  const HostT &w = T(u + ".conv_out.weight"), &bb = T(u + ".conv_out.bias"), &pq = T("vae.post_quant_conv.weight"), &pb = T("vae.post_quant_conv.bias");
  std::vector<float> f((size_t)8 * 320 * 9, 0.f);
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
  return packed.emplace("unet.tail", pack({tap_segs(f.data(), 320, 3, {320})}, 8, bias)).first->second;
}

// the decoder's conv_out averaged over its 3 output channels (the 1-channel readout)
const PackedW& WeightStore::decoder_tail1() {
  const std::string d = "vae.decoder";
  auto it = packed.find("vae.decoder.tail1");
  if (it != packed.end()) return it->second;
  const HostT &w = T(d + ".conv_out.weight"), &bb = T(d + ".conv_out.bias");
  std::vector<float> f((size_t)128 * 9, 0.f);
  for (int m = 0; m < 3; ++m)
    for (int i = 0; i < 128 * 9; ++i) f[i] += w.d[(size_t)m * 128 * 9 + i] / 3.0f;
  return packed.emplace("vae.decoder.tail1", pack({tap_segs(f.data(), 128, 3, {128})}, 1, {(bb.d[0] + bb.d[1] + bb.d[2]) / 3.0f}))
      .first->second;
}

// conv_in takes 4 channels (GenPercept, rgb_blending) or 8 = cat([rgb_latent, pred_latent]) (run.py:59-78, --archs marigold)
int WeightStore::unet_in_channels() {
  const HostT& wci = T("unet.conv_in.weight");
  GP_REQUIRE(wci.shape.size() == 4 && (wci.shape[1] == 4 || wci.shape[1] == 8), "unet.conv_in must take 4 or 8 channels");
  return (int)wci.shape[1];
}

// ------------------------------------------------------------------ CLIP text tower
const std::map<std::string, std::vector<int64_t>>& text_tower_spec() {
  static const std::map<std::string, std::vector<int64_t>> spec = [] {
    std::map<std::string, std::vector<int64_t>> s;
    const std::string m = "text.text_model.";
    const int64_t D = kTextDim, F = kTextMlp;
    s[m + "embeddings.token_embedding.weight"] = {kTextVocab, D};
    s[m + "embeddings.position_embedding.weight"] = {kTextMaxTokens, D};
    auto lin = [&](const std::string& k, int64_t out, int64_t in) { s[k + ".weight"] = {out, in}; s[k + ".bias"] = {out}; };
    auto norm = [&](const std::string& k) { s[k + ".weight"] = {D}; s[k + ".bias"] = {D}; };
    for (int i = 0; i < kTextLayers; ++i) {
      const std::string p = m + "encoder.layers." + std::to_string(i);
      for (const char* n : {"q_proj", "k_proj", "v_proj", "out_proj"}) lin(p + ".self_attn." + n, D, D);
      norm(p + ".layer_norm1");
      norm(p + ".layer_norm2");
      lin(p + ".mlp.fc1", F, D);
      lin(p + ".mlp.fc2", D, F);
    }
    norm(m + "final_layer_norm");
    return s;
  }();
  return spec;
}

// [q_proj / 8 ; k_proj ; v_proj] with the biases likewise: one token GEMM writes q | k | v, the softmax scale d^-1/2 = 1/8
// folded into the q rows (a power of two: the fold is exact)
const PackedW& WeightStore::text_qkv_w(const std::string& p) {
  auto it = packed.find(p + ".qkv");
  if (it != packed.end()) return it->second;
  const size_t DD = (size_t)kTextDim * kTextDim;
  const float scale = 1.0f / std::sqrt((float)(kTextDim / kTextHeads));
  std::vector<float> m(3 * DD), bias(3 * kTextDim);
  const char* parts[3] = {".q_proj", ".k_proj", ".v_proj"};
  for (int k = 0; k < 3; ++k) {
    const float f = k == 0 ? scale : 1.0f;
    const HostT &w = T(p + parts[k] + ".weight"), &b = T(p + parts[k] + ".bias");
    for (size_t i = 0; i < DD; ++i) m[k * DD + i] = w.d[i] * f;
    for (int i = 0; i < kTextDim; ++i) bias[k * kTextDim + i] = b.d[i] * f;
  }
  return mat_w(p + ".qkv", 3 * kTextDim, kTextDim, m.data(), bias);
}

const float* WeightStore::f32_w(const std::string& key) {
  auto it = f32s.find(key);
  if (it != f32s.end()) return it->second;
  return f32s.emplace(key, upload(T(key).d)).first->second;
}

// ------------------------------------------------------------------ timestep
void WeightStore::compute_temb(int timestep) {
  if (!temb.empty()) return;
  if (te_w1.empty()) {
    te_w1 = T("unet.time_embedding.linear_1.weight").d; te_b1 = T("unet.time_embedding.linear_1.bias").d;
    te_w2 = T("unet.time_embedding.linear_2.weight").d; te_b2 = T("unet.time_embedding.linear_2.bias").d;
  }
  temb = temb_for(timestep);
  cur_timestep = timestep;
}
std::vector<float> WeightStore::temb_for(int timestep) const {
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

// The folded conv1 bias of every time-embedded ResNet at `timestep`, in temb_layers order, computed once per timestep.
const std::vector<std::vector<float>>& WeightStore::temb_biases(int timestep) {
  GP_REQUIRE(timestep >= 0 && timestep <= 1000, "gp_set_timestep: timestep must be in [0, 1000]");
  auto it = temb_cache.find(timestep);
  if (it == temb_cache.end()) {
    const std::vector<float> emb = temb_for(timestep);
    std::vector<std::vector<float>> biases(temb_layers.size());
    parallel_for((int)temb_layers.size(), [&](int i) {
      const auto& tl = temb_layers[(size_t)i];
      std::vector<float> b = temb_proj_of(tl.w, tl.b, emb);
      for (int o = 0; o < tl.cout; ++o) b[(size_t)o] += tl.conv_bias[(size_t)o];
      biases[(size_t)i] = std::move(b);
    });
    it = temb_cache.emplace(timestep, std::move(biases)).first;
  }
  return it->second;
}

float* WeightStore::temb_bias_slot(const std::string& p, int* rows) const {
  for (const auto& tl : temb_layers)
    if (tl.key == p) { *rows = tl.cout; return tl.dev_bias; }
  return nullptr;
}

const std::vector<float>& WeightStore::temb_bias(int timestep, const std::string& p) {
  const auto& biases = temb_biases(timestep);
  for (size_t i = 0; i < temb_layers.size(); ++i)
    if (temb_layers[i].key == p) return biases[i];
  throw GpError(GP_ERR_STATE, p + " has no time-embedded bias");
}

void WeightStore::set_timestep(int timestep) {
  GP_REQUIRE(timestep >= 0 && timestep <= 1000, "gp_set_timestep: timestep must be in [0, 1000]");
  if (timestep == cur_timestep) return;
  const auto& biases = temb_biases(timestep);
  GP_CUDA(cudaDeviceSynchronize());          // nothing in flight may still read the old biases
  for (size_t i = 0; i < temb_layers.size(); ++i)
    GP_CUDA(cudaMemcpy(temb_layers[i].dev_bias, biases[i].data(), (size_t)temb_layers[i].cout * 4, cudaMemcpyHostToDevice));
  cur_timestep = timestep;
}

}  // namespace gp
