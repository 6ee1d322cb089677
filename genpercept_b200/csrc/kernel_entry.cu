// Per-kernel entry points of the C-ABI: one layer at a time on caller buffers, for the parity tests and the
// micro-benchmarks.  Weights go through a throwaway WeightStore and the ops through the Builder, so these run the
// engine's own packing and launch paths.
#include <cstring>

#include "engine.h"

using namespace gp;

namespace {

void run_all(Builder& b, cudaStream_t s) {
  for (auto& op : b.ops) GP_CUDA(op.run(s));
}

// Emits `emit`'s ops on a measuring builder to size their scratch arena, allocates it (owned by `ws`), emits them again on
// a builder over that arena and runs them once on `s`, synchronised.  External tensors are addressed relative to the
// arena's base.
template <class F>
Builder build_and_run(WeightStore& ws, cudaStream_t s, F emit) {
  Builder m(ws.bf16, true, nullptr, ws.split);
  emit(m);
  GP_REQUIRE(m.long_softmax.empty(), m.long_softmax + ": rows past " + std::to_string(kSoftmaxRowsMaxT) +
                                         " keys, more than the unfused softmax takes");
  Builder b(ws.bf16, false, reinterpret_cast<uint8_t*>(ws.device_alloc(m.arena_bytes() + 1024)), ws.split);
  emit(b);
  run_all(b, s);
  GP_CUDA(cudaStreamSynchronize(s));
  return b;
}

// mean microseconds of one pass over `b`'s ops, over `iters` passes on the default stream
double time_ops(Builder& b, int iters) {
  cudaEvent_t e0, e1;
  GP_CUDA(cudaEventCreate(&e0));
  GP_CUDA(cudaEventCreate(&e1));
  GP_CUDA(cudaEventRecord(e0, 0));
  for (int i = 0; i < iters; ++i) run_all(b, 0);
  GP_CUDA(cudaEventRecord(e1, 0));
  GP_CUDA(cudaEventSynchronize(e1));
  float ms = 0;
  GP_CUDA(cudaEventElapsedTime(&ms, e0, e1));
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  return ms * 1000.0 / iters;
}

// Fills the attention benchmarks' 16-bit operands `qk` (qk_n elements) and `vT` (vt_n) with small pseudo-random values
// (scores of order one, as in the model) rather than zeros, so the tensor cores switch as they do on real data.
void fill_attention_operands(bool bf16, void* qk, size_t qk_n, void* vT, size_t vt_n) {
  std::vector<uint16_t> pat((size_t)1 << 20);
  uint32_t x = 12345u;
  for (auto& v : pat) {
    x = x * 1664525u + 1013904223u;
    const float f = ((int)(x >> 9) - (1 << 22)) * (0.3f / (1 << 22));
    v = host_f2h(f, bf16);
  }
  for (auto [buf, n] : {std::make_pair(qk, qk_n), std::make_pair(vT, vt_n)})
    for (size_t i = 0; i < n; i += pat.size())
      GP_CUDA(cudaMemcpy(reinterpret_cast<uint16_t*>(buf) + i, pat.data(), std::min(pat.size(), n - i) * 2,
                         cudaMemcpyHostToDevice));
}

// The storage layout of a per-kernel call: GP_F16 / GP_BF16, or (where the entry point takes it) GP_F16_PAIR, the
// high-precision mode's [hi C | lo C] fp16 pairs.  Returns true for the pair layout.
bool storage_layout(int dtype, bool pair_ok, const char* fn) {
  GP_REQUIRE(dtype == GP_F16 || dtype == GP_BF16 || (pair_ok && dtype == GP_F16_PAIR),
             std::string(fn) + (pair_ok ? ": dtype must be f16, bf16 or f16 pair" : ": dtype must be f16/bf16"));
  return dtype == GP_F16_PAIR;
}

}  // namespace

extern "C" {

gp_status gp_conv2d(int dtype, const void* x, int N, int H, int W, int Cin, const float* w_host, const float* bias_host,
                    int Cout, int ks, int mode, const void* residual, int relu, void* y, int use_direct, void* stream) {
  return guarded_call([&]() {
    GP_REQUIRE(x && w_host && y && (ks == 1 || ks == 3) && mode >= 0 && mode <= 3, "gp_conv2d: bad arguments");
    const bool pair = storage_layout(dtype, true, "gp_conv2d");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    WeightStore ws(dtype == GP_BF16, pair);
    ws.put("t.weight", {Cout, Cin, ks, ks}, w_host);
    if (bias_host) ws.put("t.bias", {Cout}, bias_host);
    const auto [Ho, Wo] = conv_out_dims(mode, H, W);
    Builder b(ws.bf16, false, nullptr, ws.split);
    T4 xin = b.external(x, N, H, W, Cin);
    T4 yout = b.external(y, N, Ho, Wo, Cout);
    T4 res;
    if (residual) res = b.external(residual, N, Ho, Wo, Cout);
    if (use_direct) {
      const DirectW& dw = ws.direct_w("t", Cin);
      DirectConvParams p;
      std::memset(&p, 0, sizeof(p));
      p.in = x; p.N = N; p.H = H; p.W = W; p.Cin = Cin; p.in_cstride = (int)xin.ps(); p.in_lo = pair ? Cin : 0;
      p.w = dw.w; p.bias = dw.bias; p.res = residual;
      p.out = y; p.Ho = Ho; p.Wo = Wo; p.Cout = Cout; p.out_cstride = (int)yout.ps(); p.out_lo = pair ? Cout : 0;
      p.ks = ks;
      p.stride = (mode == 1 || mode == 2) ? 2 : 1;
      p.pad = (mode == 2) ? 0 : ks / 2;
      p.flags = (relu ? DC_RELU : 0) | (mode == 3 ? DC_UP2X : 0);
      GP_CUDA(direct_conv(p, ws.bf16, s));
    } else {
      ConvArgs c;
      c.srcs = {xin};
      c.ks = ks;
      c.mode = mode;
      if (mode == 3) {
        const std::vector<float> zb(Cout, 0.f);
        if (!bias_host) ws.put("t.bias", {Cout}, zb.data());
        c.w = &ws.conv_up_w("t");
      } else {
        c.w = &ws.conv_w("t", {Cin});
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
  return guarded_call([&]() {
    GP_REQUIRE(x && y && gamma_host && beta_host && groups >= 1 && C % groups == 0 && C % 8 == 0, "gp_groupnorm: bad arguments");
    const bool pair = storage_layout(dtype, true, "gp_groupnorm");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    WeightStore ws(dtype == GP_BF16, pair);
    ws.put("gn.weight", {C}, gamma_host);
    ws.put("gn.bias", {C}, beta_host);
    const NormW& nw = ws.norm_w("gn");
    float* ss = ws.upload(std::vector<float>((size_t)N * C * 2, 0.f));
    build_and_run(ws, s, [&](Builder& b) {
      b.gn_ss = ss;
      b.gn("gp_groupnorm", {b.external(x, N, H, W, C)}, nw, groups, eps, silu != 0, b.external(y, N, H, W, C));
    });
  });
}

gp_status gp_gn_conv3x3(int dtype, const void* x, int N, int H, int W, int Cin, int groups, const float* gamma_host,
                        const float* beta_host, float eps, int silu, const float* w_host, const float* bias_host, int Cout,
                        const void* sc_x, int Csc, const float* sc_w_host, const float* sc_b_host, const void* residual,
                        void* y, int out_f32, void* stream) {
  return guarded_call([&]() {
    GP_REQUIRE(x && w_host && y && gamma_host && beta_host, "gp_gn_conv3x3: bad arguments");
    const bool pair = storage_layout(dtype, true, "gp_gn_conv3x3");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    WeightStore ws(dtype == GP_BF16, pair);
    ws.put("t.weight", {Cout, Cin, 3, 3}, w_host);
    std::vector<float> zb(Cout, 0.f);
    ws.put("t.bias", {Cout}, bias_host ? bias_host : zb.data());
    if (sc_x) {
      GP_REQUIRE(sc_w_host != nullptr, "gp_gn_conv3x3: shortcut weights missing");
      ws.put("s.weight", {Cout, Csc, 1, 1}, sc_w_host);
      ws.put("s.bias", {Cout}, sc_b_host ? sc_b_host : zb.data());
    }
    ws.put("gn.weight", {Cin}, gamma_host);
    ws.put("gn.bias", {Cin}, beta_host);
    const NormW& nw = ws.norm_w("gn");
    float* ss = ws.upload(std::vector<float>((size_t)N * Cin * 2, 0.f));
    const PackedW& pw = sc_x ? ws.conv_w("t", {Cin}, "s", {Csc}) : ws.conv_w("t", {Cin});
    build_and_run(ws, s, [&](Builder& b) {
      b.gn_ss = ss;
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
    });
  });
}

gp_status gp_conv_groupnorm(int dtype, const void* x, int N, int H, int W, int Cin, const float* w_host, const float* bias_host,
                            int Cout, const void* skip, int Cskip, int groups, const float* gamma_host, const float* beta_host,
                            float eps, int silu, void* y_conv, void* y, void* stream) {
  return guarded_call([&]() {
    GP_REQUIRE(x && w_host && y_conv && y && gamma_host && beta_host && groups >= 1 && Cout % 8 == 0 && Cskip % 8 == 0 &&
                   (skip ? Cskip > 0 : Cskip == 0) && (Cout + Cskip) % groups == 0,
               "gp_conv_groupnorm: bad arguments");
    const bool pair = storage_layout(dtype, true, "gp_conv_groupnorm");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    WeightStore ws(dtype == GP_BF16, pair);
    ws.put("t.weight", {Cout, Cin, 3, 3}, w_host);
    std::vector<float> zb(Cout, 0.f);
    ws.put("t.bias", {Cout}, bias_host ? bias_host : zb.data());
    const int Ctot = Cout + Cskip;
    ws.put("gn.weight", {Ctot}, gamma_host);
    ws.put("gn.bias", {Ctot}, beta_host);
    const NormW& nw = ws.norm_w("gn");
    float* ss = ws.upload(std::vector<float>((size_t)N * Ctot * 2, 0.f));
    const PackedW& pw = ws.conv_w("t", {Cin});
    build_and_run(ws, s, [&](Builder& b) {
      b.gn_ss = ss;
      ConvArgs c;
      c.srcs = {b.external(x, N, H, W, Cin)};
      c.w = &pw;
      c.out = b.external(y_conv, N, H, W, Cout);
      c.want_stats = true;
      b.conv("gp_conv_groupnorm.conv", c);
      std::vector<T4> srcs = {c.out};
      if (skip) srcs.push_back(b.external(skip, N, H, W, Cskip));
      b.gn("gp_conv_groupnorm.gn", srcs, nw, groups, eps, silu != 0, b.external(y, N, H, W, Ctot));
    });
  });
}

gp_status gp_layernorm(int dtype, const void* x, int64_t tokens, int C, const float* gamma_host, const float* beta_host,
                       float eps, void* y, void* stream) {
  return guarded_call([&]() {
    GP_REQUIRE(x && y && gamma_host && beta_host && tokens >= 0 && C >= 8, "gp_layernorm: bad arguments");
    const bool pair = storage_layout(dtype, true, "gp_layernorm");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    WeightStore ws(dtype == GP_BF16, pair);
    float* g = ws.upload(std::vector<float>(gamma_host, gamma_host + C));
    float* bt = ws.upload(std::vector<float>(beta_host, beta_host + C));
    GP_CUDA(layernorm(x, y, tokens, C, g, bt, eps, ws.bf16, s, pair));
    GP_CUDA(cudaStreamSynchronize(s));
  });
}

gp_status gp_attention(int dtype, const void* q, const void* k, const void* v, int B, int T, int heads, int d, float scale,
                       void* o, void* stream) {
  return guarded_call([&]() {
    // q is pre-scaled by the caller-visible `scale` through an identity-weight GEMM, and V^T is the engine's own
    // swapped-operand GEMM with identity weights, so that the same igemm paths the engine uses (QK^T, softmax, V^T, PV)
    // are exercised.
    storage_layout(dtype, false, "gp_attention");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    WeightStore ws(dtype == GP_BF16);
    const int C = heads * d;
    std::vector<float> eye((size_t)C * C, 0.f), eyes((size_t)C * C, 0.f);
    for (int i = 0; i < C; ++i) { eye[(size_t)i * C + i] = 1.f; eyes[(size_t)i * C + i] = scale; }
    const PackedW& wv = ws.mat_w("eye", C, C, eye.data(), {});
    const PackedW& wq = ws.mat_w("eyes", C, C, eyes.data(), {});
    const int Tp = ceil_div(T, 8) * 8;
    void* qs = ws.device_alloc((size_t)B * T * C * 2);
    void* vT = ws.device_alloc((size_t)B * C * Tp * 2);
    build_and_run(ws, s, [&](Builder& b) {
      { ConvArgs c; c.srcs = {b.external(q, B, 1, T, C)}; c.ks = 1; c.w = &wq; c.out = b.external(qs, B, 1, T, C); b.conv("scale_q", c); }
      b.to_vT("v", b.external(v, B, 1, T, C), wv, vT);
      b.attention_qkv("attn", qs, k, C, vT, B, T, heads, d, nullptr, b.external(o, B, 1, T, C));
    });
  });
}

gp_status gp_attention_high(const void* qk, const void* v, int B, int T, int heads, int d, int fused, void* o, void* stream) {
  return guarded_call([&]() {
    GP_REQUIRE(qk && v && o && B >= 1 && T >= 1 && (d == 64 || (d == 512 && heads == 1)),
               "gp_attention_high: bad arguments (d = 64, or d = 512 with one head)");
    // V^T is the engine's swapped-operand GEMM with identity weights (hi 1, lo 0), which reproduces v's (hi, lo) pairs
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    WeightStore ws(false, true);
    const int C = heads * d;
    const int Tp = ceil_div(T, 8) * 8;
    std::vector<float> eye((size_t)C * C, 0.f);
    for (int i = 0; i < C; ++i) eye[(size_t)i * C + i] = 1.f;
    const PackedW& wv = ws.mat_w("eye", C, C, eye.data(), {});
    void* vT = ws.device_alloc((size_t)B * C * 2 * Tp * 2);
    build_and_run(ws, s, [&](Builder& b) {
      b.mem_efficient_attn = fused != 0;
      b.to_vT("v", b.external(v, B, 1, T, C), wv, vT);
      const uint16_t* q = reinterpret_cast<const uint16_t*>(qk);
      b.attention_qkv("attn", q, q + C, 4LL * C, vT, B, T, heads, d, nullptr, b.external(o, B, 1, T, C), 2LL * C);
    });
  });
}

gp_status gp_ensemble_reduce(const float* pred_dev, int B, int H, int W, const float* scale_host, const float* shift_host,
                             int median, int normalise, float* out_dev, void* stream) {
  return guarded_call([&]() {
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
  return guarded_call([&]() {
    GP_REQUIRE(x && y && N >= 1 && H >= 1 && W >= 1 && C >= 1, "gp_bilinear_up2x: bad arguments");
    const bool pair = storage_layout(dtype, true, "gp_bilinear_up2x");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    GP_CUDA(bilinear_up2x(x, y, N, H, W, C, dtype == GP_BF16, s, pair));
    GP_CUDA(cudaStreamSynchronize(s));
  });
}

gp_status gp_geglu(int dtype, const void* x, int64_t tokens, int C, const float* w_host, const float* b_host, void* y,
                   void* stream) {
  return guarded_call([&]() {
    GP_REQUIRE(x && y && w_host && b_host && tokens >= 1 && tokens < (1LL << 31) && C >= 8 && C % 8 == 0,
               "gp_geglu: bad arguments (C % 8 == 0)");
    const bool pair = storage_layout(dtype, true, "gp_geglu");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    WeightStore ws(dtype == GP_BF16, pair);
    ws.put("t.ff.net.0.proj.weight", {8LL * C, C}, w_host);
    ws.put("t.ff.net.0.proj.bias", {8LL * C}, b_host);
    build_and_run(ws, s, [&](Builder& b) {
      geglu_projection(b, ws, "t", b.external(x, 1, 1, (int)tokens, C), b.external(y, 1, 1, (int)tokens, 4 * C));
    });
  });
}

gp_status gp_cross_attention(int dtype, const void* x, int64_t tokens, int C, int heads, const float* ctx_host, int n, int E,
                             const float* to_q, const float* to_k, const float* to_v, const float* to_out_w,
                             const float* to_out_b, const float* norm_g, const float* norm_b, float eps, void* y,
                             void* stream) {
  return guarded_call([&]() {
    GP_REQUIRE(x && y && ctx_host && to_q && to_k && to_v && to_out_w && to_out_b && norm_g && norm_b && tokens >= 1 &&
                   tokens < (1LL << 31) && heads >= 1 && C % heads == 0 && C % 8 == 0 && n >= 1 && E >= 1,
               "gp_cross_attention: bad arguments (C % 8 == 0, C % heads == 0)");
    const bool pair = storage_layout(dtype, true, "gp_cross_attention");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    WeightStore ws(dtype == GP_BF16, pair);
    ws.text_embed.assign(ctx_host, ctx_host + (size_t)n * E);
    ws.n_tokens = n;
    ws.put("t.attn2.to_q.weight", {C, C}, to_q);
    ws.put("t.attn2.to_k.weight", {C, E}, to_k);
    ws.put("t.attn2.to_v.weight", {C, E}, to_v);
    ws.put("t.attn2.to_out.0.weight", {C, C}, to_out_w);
    ws.put("t.attn2.to_out.0.bias", {C}, to_out_b);
    ws.put("t.norm2.weight", {C}, norm_g);
    ws.put("t.norm2.bias", {C}, norm_b);
    build_and_run(ws, s, [&](Builder& b) {
      const int T = (int)tokens;
      cross_attention(b, ws, "t", b.external(x, 1, 1, T, C), heads, eps, b.external(y, 1, 1, T, C));
    });
  });
}

gp_status gp_resnet(int dtype, const void* x, int Cx, const void* skip, int Cskip, int N, int H, int W, int Cout, float eps,
                    const float* norm1_g, const float* norm1_b, const float* conv1_w, const float* conv1_b,
                    const float* norm2_g, const float* norm2_b, const float* conv2_w, const float* conv2_b,
                    const float* shortcut_w, const float* shortcut_b, void* y, void* stream) {
  return guarded_call([&]() {
    const int Cin = Cx + Cskip;
    GP_REQUIRE(x && y && norm1_g && norm1_b && conv1_w && conv1_b && norm2_g && norm2_b && conv2_w && conv2_b && N >= 1 &&
                   H >= 1 && W >= 1 && Cx >= 8 && Cx % 8 == 0 && Cskip % 8 == 0 && (skip ? Cskip > 0 : Cskip == 0) &&
                   Cin % 32 == 0 && Cout >= 32 && Cout % 32 == 0,
               "gp_resnet: bad arguments (channels: multiples of 8, Cx + Cskip and Cout of 32)");
    GP_REQUIRE((shortcut_w && shortcut_b) == (Cin != Cout) && (shortcut_w != nullptr) == (shortcut_b != nullptr),
               "gp_resnet: the shortcut weights are required exactly when Cx + Cskip != Cout");
    const bool pair = storage_layout(dtype, true, "gp_resnet");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    WeightStore ws(dtype == GP_BF16, pair);
    ws.put("t.norm1.weight", {Cin}, norm1_g);
    ws.put("t.norm1.bias", {Cin}, norm1_b);
    ws.put("t.conv1.weight", {Cout, Cin, 3, 3}, conv1_w);
    ws.put("t.conv1.bias", {Cout}, conv1_b);
    ws.put("t.norm2.weight", {Cout}, norm2_g);
    ws.put("t.norm2.bias", {Cout}, norm2_b);
    ws.put("t.conv2.weight", {Cout, Cout, 3, 3}, conv2_w);
    ws.put("t.conv2.bias", {Cout}, conv2_b);
    if (shortcut_w) {
      ws.put("t.conv_shortcut.weight", {Cout, Cin, 1, 1}, shortcut_w);
      ws.put("t.conv_shortcut.bias", {Cout}, shortcut_b);
    }
    float* ss = ws.upload(std::vector<float>((size_t)N * std::max(Cin, Cout) * 2, 0.f));
    build_and_run(ws, s, [&](Builder& b) {
      b.gn_ss = ss;
      std::vector<T4> xs = {b.external(x, N, H, W, Cx)};
      if (skip) xs.push_back(b.external(skip, N, H, W, Cskip));
      const T4 out = resnet_block(b, ws, "t", xs, Cout, eps, false);
      // the block writes a tensor of the arena; the caller's y takes a copy
      if (!b.measuring()) {
        const void* src = b.ptr(out);
        const size_t nb = out.bytes();
        b.custom("gp_resnet.out", 1, 2.0 * nb,
                 [=](cudaStream_t st) { return cudaMemcpyAsync(y, src, nb, cudaMemcpyDeviceToDevice, st); });
      }
      b.release(out);
    });
  });
}

gp_status gp_resize(int dtype, const void* x, int N, int H, int W, int C, int OH, int OW, int mode, void* y, void* stream) {
  return guarded_call([&]() {
    GP_REQUIRE(x && y && N >= 1 && H >= 1 && W >= 1 && OH >= 1 && OW >= 1 && C >= 8 && C % 8 == 0 && (mode == 0 || mode == 1),
               "gp_resize: bad arguments (C % 8 == 0, mode 0 nearest or 1 bilinear)");
    const bool pair = storage_layout(dtype, true, "gp_resize");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    WeightStore ws(dtype == GP_BF16, pair);
    build_and_run(ws, s, [&](Builder& b) {
      b.resize("gp_resize", b.external(x, N, H, W, C), b.external(y, N, OH, OW, C), mode == 0);
    });
  });
}

gp_status gp_causal_attention(int dtype, const void* qkv, int n, int heads, int d, void* out, void* stream) {
  return guarded_call([&]() {
    GP_REQUIRE(qkv && out && n >= 1 && n <= kTextMaxTokens && heads >= 1 && d >= 1 && d <= kCausalMaxD,
               "gp_causal_attention: bad arguments (1 <= n <= 77, 1 <= d <= 64)");
    const bool pair = storage_layout(dtype, true, "gp_causal_attention");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    GP_CUDA(causal_attention(qkv, n, heads, d, out, dtype == GP_BF16, s, pair));
    GP_CUDA(cudaStreamSynchronize(s));
  });
}

gp_status gp_gelu(int dtype, const void* x, int64_t n_elems, void* y, void* stream) {
  return guarded_call([&]() {
    GP_REQUIRE(x && y && n_elems >= 8 && n_elems % 8 == 0 && n_elems < (1LL << 30), "gp_gelu: bad arguments (n_elems % 8 == 0)");
    const bool pair = storage_layout(dtype, true, "gp_gelu");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    GP_CUDA(gelu16(x, y, n_elems, dtype == GP_BF16, s, pair ? (int)n_elems : 0));
    GP_CUDA(cudaStreamSynchronize(s));
  });
}

gp_status gp_bench_conv(int dtype, int N, int H, int W, int Cin, int Cout, int ks, int mode, int iters, double* usec,
                        double* flops) {
  return guarded_call([&]() {
    storage_layout(dtype, false, "gp_bench_conv");
    WeightStore ws(dtype == GP_BF16);
    const std::vector<float> wt((size_t)Cout * Cin * ks * ks, 0.01f), bz(Cout, 0.f);
    ws.put("t.weight", {Cout, Cin, ks, ks}, wt.data());
    ws.put("t.bias", {Cout}, bz.data());
    const auto [Ho, Wo] = conv_out_dims(mode, H, W);
    void* x = ws.device_alloc((size_t)N * H * W * Cin * 2);
    void* y = ws.device_alloc((size_t)N * Ho * Wo * Cout * 2);
    GP_CUDA(cudaMemset(x, 0, (size_t)N * H * W * Cin * 2));
    Builder b(ws.bf16, false, nullptr);
    ConvArgs c;
    c.srcs = {b.external(x, N, H, W, Cin)};
    c.ks = ks; c.mode = mode;
    c.w = (mode == 3) ? &ws.conv_up_w("t") : &ws.conv_w("t", {Cin});
    c.out = b.external(y, N, Ho, Wo, Cout);
    b.conv("bench", c);
    for (int i = 0; i < 3; ++i) run_all(b, 0);
    const double us = time_ops(b, iters);
    if (usec) *usec = us;
    if (flops) *flops = b.ops[0].flops;
  });
}

gp_status gp_bench_attention(int dtype, int B, int T, int fused, int iters, double* usec, double* flops) {
  return guarded_call([&]() {
    storage_layout(dtype, false, "gp_bench_attention");
    GP_REQUIRE(B >= 1 && T >= 1 && iters >= 1, "gp_bench_attention: bad arguments");
    WeightStore ws(dtype == GP_BF16);
    const int C = 512;
    const int Tp = ceil_div(T, 8) * 8;
    // The VAE mid-block's operands: q | k packed at a pixel stride of 2C, V^T [B][C][Tp], out [B][T][C].
    const size_t qk_n = (size_t)B * T * 2 * C, vt_n = (size_t)B * C * Tp, o_n = (size_t)B * T * C;
    void* qk = ws.device_alloc(qk_n * 2);
    void* vT = ws.device_alloc(vt_n * 2);
    void* o = ws.device_alloc(o_n * 2);
    fill_attention_operands(ws.bf16, qk, qk_n, vT, vt_n);
    // one warm-up launch, synchronised
    Builder b = build_and_run(ws, 0, [&](Builder& bb) {
      bb.attn512_path = fused ? 1 : 0;
      bb.attention_qkv("attn", qk, reinterpret_cast<uint16_t*>(qk) + C, 2 * C, vT, B, T, 1, C, nullptr,
                       bb.external(o, B, 1, T, C));
    });
    const double us = time_ops(b, iters);
    if (usec) *usec = us;
    if (flops) *flops = 4.0 * B * (double)T * T * C;
  });
}

gp_status gp_bench_attention_high(int B, int T, int heads, int d, int fused, int iters, double* usec, double* flops) {
  return guarded_call([&]() {
    GP_REQUIRE(B >= 1 && T >= 1 && iters >= 1 && (d == 64 || (d == 512 && heads == 1)),
               "gp_bench_attention_high: bad arguments (d = 64, or d = 512 with one head)");
    WeightStore ws(false, true);
    const int C = heads * d;
    const int Tp = ceil_div(T, 8) * 8;
    // the engine's operands: [q hi | k hi | q lo | k lo] per token, V^T [B][C][hi Tp | lo Tp], out [B][T][hi C | lo C]
    const size_t qk_n = (size_t)B * T * 4 * C, vt_n = (size_t)B * C * 2 * Tp, o_n = (size_t)B * T * 2 * C;
    void* qk = ws.device_alloc(qk_n * 2);
    void* vT = ws.device_alloc(vt_n * 2);
    void* o = ws.device_alloc(o_n * 2);
    fill_attention_operands(false, qk, qk_n, vT, vt_n);     // lo planes included
    // one warm-up launch, synchronised
    Builder b = build_and_run(ws, 0, [&](Builder& bb) {
      bb.mem_efficient_attn = fused != 0;
      const uint16_t* q = reinterpret_cast<const uint16_t*>(qk);
      bb.attention_qkv("attn", q, q + C, 4LL * C, vT, B, T, heads, d, nullptr, bb.external(o, B, 1, T, C), 2LL * C);
    });
    const double us = time_ops(b, iters);
    if (usec) *usec = us;
    if (flops) *flops = 4.0 * B * heads * (double)T * T * d;
  });
}

}  // extern "C"
