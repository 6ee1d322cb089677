/* genpercept_b200 — C-ABI of the H100-native one-step perception engine.
 *
 * This is the drop-in boundary for the hot path of aim-uofa/GenPercept:
 *   GenPerceptPipeline.single_infer        /root/reference/genpercept/genpercept_pipeline.py:375-486
 *     encode_rgb  (vae.encoder, quant_conv, mean * 0.18215)                     :488-505
 *     unet(pred_latent, t=1, empty-text embed) + DDIM(beta=1) step == -v       :443-465
 *     decode_pred (/0.18215, post_quant_conv, vae.decoder, channel mean)       :507-526
 *     clip(-1,1), (x+1)/2                                                      :470-472
 *     or the DPT readout (customized_head on multi_level_feats, min-max)       :475-482
 * Everything below the boundary is hand-written sm_90a CUDA; there is no CPU fallback: every
 * entry point returns GP_ERR_CUDA when no CUDA device / kernel image is available.
 *
 * Plain C types only.  Device pointers are raw CUdeviceptr-compatible addresses (e.g.
 * torch.Tensor.data_ptr()); `stream` is a cudaStream_t passed as void*.
 */
#ifndef GENPERCEPT_B200_H
#define GENPERCEPT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct gp_engine gp_engine;

typedef enum {
  GP_OK = 0,
  GP_ERR_INVALID = 1,   /* bad argument / shape (reference: Python assert / ValueError) */
  GP_ERR_MISSING = 2,   /* a checkpoint tensor required by the topology was never loaded  */
  GP_ERR_NO_PLAN = 3,   /* gp_infer before gp_plan for this (B,H,W)                        */
  GP_ERR_CUDA = 4,      /* CUDA error (sticky: the engine is poisoned)                      */
  GP_ERR_STATE = 5      /* call order (e.g. gp_plan before gp_finalize)                     */
} gp_status;

/* GP_F16_PAIR: the high-precision mode's storage layout (gp_config.precision = 1), taken by the per-kernel entry points
 * that say so: a 16-bit tensor of C logical channels carries [hi C | lo C] fp16 per pixel, value = hi + lo.  Every other
 * entry point rejects it with GP_ERR_INVALID. */
typedef enum { GP_F32 = 0, GP_F16 = 1, GP_BF16 = 2, GP_U8 = 3, GP_F16_PAIR = 4 } gp_dtype;
typedef enum { GP_READOUT_VAE = 0, GP_READOUT_DPT = 1 } gp_readout;

typedef struct {
  int device;            /* CUDA device ordinal                                             */
  int dtype;             /* GP_F16 or GP_BF16: storage / tensor-core operand type            */
  int readout;           /* gp_readout: VAE decoder (run.py default) or DPT head (:296-301)  */
  int timestep;          /* UNet timestep; 1 for GenPercept (ddim.py + scheduler beta=1), or
                            the reference's --fix_timesteps value                           */
  int use_cuda_graph;    /* 0 eager, 1 replay one captured CUDA graph per plan, 2 auto (small plans) */
  int precision;         /* 0: 16-bit storage, fp32 accumulate (the reference's --half_precision class);
                            1: high — every activation and weight is carried as an fp16 (hi, lo) pair and every
                            contraction runs hi*hi + lo*hi + hi*lo on the tensor cores (fp32-class products,
                            fp32 accumulate): the reference's default fp32 run (run.py:273-281)              */
  int arch;              /* 0: one-step GenPercept (the scheduler's beta = 1 step folded into the UNet tail);
                            1: multi-step (run.py --archs marigold / rgb_blending): the UNet returns model_output, real
                            DDIM steps run around it (gp_infer_steps); conv_in may take 8 channels (run.py:59-78)   */
} gp_config;

/* replaces: GenPerceptPipeline.__init__/from_pretrained model assembly (run.py:314-376) */
gp_status gp_create(const gp_config* cfg, gp_engine** out);
void gp_destroy(gp_engine* e);
/* the reason of engine `e`'s last failed call */
const char* gp_last_error(gp_engine* e);
/* the reason of the calling thread's last failed call that takes no engine (gp_create, the per-kernel, pre/post,
 * evaluation, JPEG, shared-arena and host-only query entry points), or "" when the last such call succeeded */
const char* gp_last_call_error(void);

/* replaces: load_state_dict of the diffusers-format checkpoints (run.py:336-357, :296-312).
 * `key` = "<component>.<diffusers key>", component in {unet, vae, dpt}, or "text" (gp_encode_text).  Host pointer, copied. */
gp_status gp_load_tensor(gp_engine* e, const char* key, const void* host_ptr, int dtype,
                         const int64_t* shape, int ndim);
/* replaces: encode_text()'s cached self.text_embed (genpercept_pipeline.py:360-372, :425-429).
 * fp32 [n_tokens, 1024].  n_tokens == 2 (the empty prompt) takes the closed-form cross-attention; any other
 * length the general one (context projections folded into two 1x1 GEMMs around a per-head softmax).  The
 * context is a constant of the engine from gp_finalize on, like the reference's cached self.text_embed. */
gp_status gp_set_text_embed(gp_engine* e, const float* host_ptr, int n_tokens, int dim);
/* replaces: encode_text()'s text_encoder(text_input_ids)[0] (genpercept_pipeline.py:360-372), SD-2.1's CLIPTextModel, on
 * the engine in its mode (16-bit, or the high-precision pair layout).  ids_host: n_tokens token ids (int32, host) as the
 * tokenizer gives them, 1 <= n_tokens <= 77, each in [0, 49408); out_host: fp32 [n_tokens, 1024] = last_hidden_state after
 * final_layer_norm, ready for gp_set_text_embed.  Its weights are gp_load_tensor's component "text": "text." + the
 * CLIPTextModel state-dict keys ("text.text_model.encoder.layers.0.self_attn.q_proj.weight", ...; the position_ids buffer
 * is ignored), each checked against SD-2.1's shapes on load (GP_ERR_INVALID otherwise, e.g. SD-1.x's d = 768 tower).  The
 * tower packs its own weights and an arena per n_tokens on first use, apart from the image plans (gp_plan_info's weight
 * bytes do not count them), and runs on `stream`; it returns after the copy.  Errors leave the engine usable: a bad id or
 * n_tokens GP_ERR_INVALID, a text tensor never loaded GP_ERR_MISSING, a call after gp_finalize GP_ERR_STATE. */
gp_status gp_encode_text(gp_engine* e, const int32_t* ids_host, int n_tokens, float* out_host, void* stream);
/* folds constants (SURVEY.md App. C), re-packs weights K-major 16-bit, uploads.  Frees the text tower's host tensors,
 * device weights and arenas: from here on the context is a constant of the engine. */
gp_status gp_finalize(gp_engine* e);

/* builds the static op list, activation arena and (optionally) CUDA graph for one input shape.  Any H, W >= 32: the
 * result extent (gp_tensor_shape "out") is 8*floor(H/8) x 8*floor(W/8) for the VAE readout (AutoencoderKL's
 * stride-2 stages floor) and the DPT head's pyramid extent for the DPT readout; equal to H x W for multiples of 8 / 64. */
gp_status gp_plan(gp_engine* e, int batch, int height, int width);

/* number of cached plans (the cache is bounded: least-recently-used plans are destroyed; GP_MAX_PLANS, default 4) */
int gp_plan_count(gp_engine* e);
/* replaces: pipe.enable_xformers_memory_efficient_attention() / disable_... (run.py:382-385, infer.py:400-403).
 * enable != 0: in the high-precision mode (gp_config.precision = 1) every self-attention (head_dim 64) and VAE mid-block
 * attention (head_dim 512) runs fused, so no T x T score matrix is stored and a plan's memory grows with the pixel count.
 * Off by default: the high-precision plans then store the score matrices, and a shape whose rows exceed the unfused
 * softmax's 16384 keys fails at gp_plan with GP_ERR_INVALID.  The 16-bit modes always bound the score matrix and ignore
 * the switch.  Valid before or after gp_finalize; a change of value drops the cached plans. */
gp_status gp_set_memory_efficient_attention(gp_engine* e, int enable);
/* One activation arena per device for the engines that opt in, as PyTorch's caching allocator serves every pipeline of a
 * process in the reference.  enable != 0: this engine's plans take their arena from the device's shared pool instead of
 * a cudaMalloc of their own, so N engines (or N cached plans) need the largest arena among them, not the sum.  The pool
 * reserves a virtual range the size of the device's memory once and maps physical memory behind a fixed base: it grows
 * when a larger plan is made, shrinks (after a device synchronisation) when the largest plan goes, and unmaps everything
 * when the last engine using it leaves.  A plan that does not fit fails at gp_plan with GP_ERR_INVALID, as without the
 * pool, and the engine stays usable.  Every call that touches a shared plan's arena waits on the pool's one event on its
 * stream first and records it after its last operation, so engines on different streams take turns without a host
 * synchronisation.  Off by default (every path, op list, arena size and result is then as without the pool).  Valid
 * before or after gp_finalize; a change of value synchronises and drops the cached plans.
 * Semantics of a shared plan:
 *   - its kept tensors ("rgb_latent", "z", "feat0".., "out" of gp_read_tensor) hold meaningful data only until another
 *     plan in the pool runs or the pool shrinks, so gp_run_stage chains and gp_read_tensor are meaningful only straight
 *     after the plan's own call;
 *   - results always leave through the caller's buffer, as without the pool;
 *   - one host thread per pool: concurrent host threads on the engines of one device are not supported. */
gp_status gp_set_shared_arena(gp_engine* e, int enable);
/* The device's shared pool: bytes mapped now (the largest live shared plan's arena rounded up to the allocation
 * granularity), bytes of virtual address space reserved, and the number of live plans in it; all 0 when no engine on
 * `device` shares it. */
gp_status gp_shared_arena_info(int device, int64_t* mapped_bytes, int64_t* reserved_bytes, int64_t* live_plans);
/* Tests: writes `byte` over the whole mapped range on `stream`, ordered after every earlier user of the pool and before
 * every later one.  No op reads arena bytes it did not write in the same call, so results do not change.  GP_ERR_STATE
 * when no engine on `device` shares the pool. */
gp_status gp_shared_arena_fill(int device, int byte, void* stream);
/* Host-only introspection (no device needed): the N tile (BN) and the number of 128-pixel M tiles per CTA (MT) the planner
 * gives a stride-1 ks x ks convolution / linear layer cin -> cout over `images` maps of h x w output pixels on a GPU with
 * num_sms SMs (tokens_mode != 0: one row of images * h * w tokens).  Nothing in the reference corresponds to it (PyTorch /
 * cuDNN pick their own tiles); it pins the tile policy of tile_shape_for (csrc/builder.cu) in the CPU tests. */
gp_status gp_tile_shape(int cout, int cin, int ks, int images, int h, int w, int tokens_mode, int num_sms, int* bn, int* mt);
/* Host-only introspection: the tile the planner gives a 3x3 stride-1 convolution cin -> cout (plus a fused 1x1 shortcut over
 * csc channels, or 0) over `images` maps of h x w pixels in the 16-bit modes: (BN, MT) as gp_tile_shape, and patch = 1 when
 * it runs on the patch-resident kernel (16 x 8 MT pixel tiles), 0 for the tap-streaming kernel. */
gp_status gp_conv_tile(int cin, int csc, int cout, int images, int h, int w, int num_sms, int* bn, int* mt, int* patch);
/* replaces: the per-call `fix_timesteps` of single_infer (/root/reference/genpercept/genpercept_pipeline.py:405-408).
 * The timestep only enters through conv1.bias + time_emb_proj(silu(emb(t))) of the 22 UNet ResNets; those biases are
 * re-folded on the host (cached per timestep) and rewritten in place after a device synchronisation. */
gp_status gp_set_timestep(gp_engine* e, int timestep);
/* Host-only: the layout of one step's row of gp_infer_steps' bias table, one segment per time-embedded UNet ResNet
 * (down blocks, mid block, up blocks): its offset and length in floats.  *n_segments gets the count (22); offsets and
 * lengths (nullable) need `capacity` >= that count. */
gp_status gp_step_bias_layout(int capacity, int* n_segments, int* offsets, int* lengths);

/* replaces: single_infer.  rgb: [B,3,H,W] NCHW, device (or pinned/pageable host if
 * rgb_on_host != 0; copied on `stream`), dtype GP_U8 (0..255, mapped x/255*2-1 as
 * genpercept_pipeline.py:245) or GP_F16/GP_F32 already in [-1,1].
 * out: fp32 [B,C,outH,outW] in [0,1] (a device `out` is written by the last kernel itself), C = out_channels (1: channel-mean modes depth/matting/dis/
 * disparity :523-525; 3: normal/seg); device, or host if out_on_host != 0.  Asynchronous on
 * `stream` unless a host buffer is involved, in which case it returns after the copy. */
gp_status gp_infer(gp_engine* e, const void* rgb, int rgb_dtype, int rgb_on_host, float* out,
                   int out_on_host, int out_channels, void* stream);

/* replaces: encode_rgb (/root/reference/genpercept/genpercept_pipeline.py:488-505).  rgb as for gp_infer; latent_dev:
 * fp32 [B,4,H/8,W/8] on the device = mean(quant_conv(encoder(rgb))) * 0.18215. */
gp_status gp_encode(gp_engine* e, const void* rgb, int rgb_dtype, int rgb_on_host, float* latent_dev, void* stream);
/* replaces: decode_pred + clip + shift (:507-526, :470-472).  latent_dev: fp32 [B,4,h,w] on the device (in the scaled
 * latent space, like the reference's pred_latent); apply_post_quant != 0 applies vae.post_quant_conv to latent / 0.18215 as
 * the reference always does (0: the latent already went through it, e.g. the engine's own "z").  out_dev: fp32
 * [B,C,8h,8w] in [0,1] (the reference clips to [-1,1] right after decode_pred, :470; map = out * 2 - 1). */
gp_status gp_decode(gp_engine* e, const float* latent_dev, int apply_post_quant, float* out_dev, int out_channels, void* stream);
/* replaces: encode_rgb for a hand-off to gp_infer_latent: the latent exactly as the plan holds it.  16-bit modes: fp32
 * [B,4,H/8,W/8], the same as gp_encode.  High-precision mode (gp_config.precision = 1): fp32 [B,8,H/8,W/8] = [hi 0..3 |
 * lo 0..3], the (hi, lo) fp16 pair of every value.  gp_encode's fp32 hi + lo does not determine the pair: where lo
 * rounded to half an ulp of hi, splitting the sum again ties to even and can pick the other neighbour. */
gp_status gp_encode_exact(gp_engine* e, const void* rgb, int rgb_dtype, int rgb_on_host, float* latent_dev, void* stream);
/* replaces: single_infer from rgb_latent on (genpercept_pipeline.py:411-486) for a latent gp_encode_exact produced, on this
 * or on another engine with the same dtype, precision and VAE encoder (several task engines share one encode).
 * latent_dev: [batch, channels, height, width] on the device as gp_encode_exact writes it (channels 4, or 8 in the
 * high-precision mode); it must match the current plan's "rgb_latent": gp_plan(B,H,W) for the image it came from (the
 * latent's extent alone does not fix the image's, which sets the DPT readout's and the result's extent), else
 * GP_ERR_INVALID.  Runs the plan's UNet and readout ops (GP_STAGE_UNET .. GP_STAGE_READOUT), with their own CUDA graph
 * when the plan uses graphs; gp_infer's graph is left as it is.  The maps equal gp_infer's on the same image bit for bit.
 * out, out_on_host, out_channels: as gp_infer.  One-step arch only (gp_config.arch = 0; else GP_ERR_INVALID). */
gp_status gp_infer_latent(gp_engine* e, const float* latent_dev, int batch, int channels, int height, int width, float* out,
                          int out_on_host, int out_channels, void* stream);

/* replaces: single_infer for the multi-step archs (/root/reference/genpercept/genpercept_pipeline.py:399-472; gp_config.arch = 1):
 *   rgb_latent = encode_rgb(rgb); pred_latent = noise (marigold; fp32 [B,4,h,w], host or device) or rgb_latent (noise == NULL:
 *   rgb_blending); per step i: unet(cat([rgb_latent, pred_latent]) or pred_latent, timesteps[i]) -> DDIM step with
 *   coeffs[4 i .. 4 i + 3] = (x0 <- sample, x0 <- model_output, prev <- sample, prev <- model_output) (eta = 0; host
 *   arrays, genpercept_b200/scheduler.py); then decode_pred(pred_original_sample), clip, shift.  out as for gp_infer.
 * Each step's conv1 biases (folded on the host, cached per timestep) and coefficients are uploaded with the call on
 * `stream` and copied into place on the device before the step, so no host or device synchronisation runs between
 * steps.  With CUDA graphs on (gp_config.use_cuda_graph, the same rule as gp_infer), the first call for each
 * (n_steps, noise given or not, out_channels) runs eagerly and later calls replay one graph of the whole loop, encode to
 * readout.  Asynchronous on `stream` unless a host buffer is involved, in which case it returns after the copy.  After the
 * call the UNet holds the last step's timestep (as gp_set_timestep(timesteps[n_steps - 1]) would leave it). */
gp_status gp_infer_steps(gp_engine* e, const void* rgb, int rgb_dtype, int rgb_on_host, const float* noise, int noise_on_host,
                         const int* timesteps, const float* coeffs, int n_steps, float* out, int out_on_host, int out_channels,
                         void* stream);

/* Stage entry points for parity tests (each runs a contiguous slice of the planned op list). */
typedef enum { GP_STAGE_PRE = 0, GP_STAGE_VAE_ENCODE = 1, GP_STAGE_UNET = 2, GP_STAGE_READOUT = 3 } gp_stage;
gp_status gp_run_stage(gp_engine* e, int stage, int out_channels, void* stream);
/* Named internal tensors kept alive by the plan: "rgb", "rgb_latent", "z" (decoder input =
 * post_quant_conv(-unet_out/0.18215)), "feat0".."feat3" (DPT taps), "out".  fp32 NCHW on host. */
gp_status gp_tensor_shape(gp_engine* e, const char* name, int64_t shape[4]);
gp_status gp_read_tensor(gp_engine* e, const char* name, float* host_out, size_t capacity_elems);
gp_status gp_write_tensor(gp_engine* e, const char* name, const float* host_in, size_t elems);

/* Introspection for bench.py */
gp_status gp_plan_info(gp_engine* e, int64_t* n_ops, int64_t* n_kernel_launches, int64_t* arena_bytes,
                       int64_t* weight_bytes, double* igemm_flops);
/* name/us of the i-th op after gp_profile_ops ran the plan once with CUDA events per op. */
gp_status gp_profile_ops(gp_engine* e, int out_channels, void* stream);
/* kind: 1 = wgmma implicit-GEMM launch, 2 = fused attention, 0 = other kernels.  flops = algorithmic work of the op
 * (SURVEY.md 8d); flops_exec = MMA work actually issued (differs for the upsample-fused convolutions: 4 of 9 taps). */
gp_status gp_op_info(gp_engine* e, int64_t i, char* name_buf, size_t name_cap, double* usec, double* flops,
                     double* bytes, int* kind, double* flops_exec);

/* ---- per-kernel entry points (parity tests, micro-benchmarks); all pointers are device ----
 * dtype: GP_F16 or GP_BF16; gp_conv2d, gp_groupnorm, gp_gn_conv3x3, gp_conv_groupnorm, gp_layernorm,
 * gp_bilinear_up2x and the UNet block ops (gp_geglu .. gp_resize) also take GP_F16_PAIR, in which every 16-bit tensor (inputs, residual, skip, shortcut, outputs) has
 * the [hi C | lo C] layout and the contractions run the high-precision mode's three passes (hi*hi + lo*hi + hi*lo). */
/* 3x3 / 1x1 convolution through the wgmma implicit-GEMM kernels.  x: 16-bit NHWC [N,H,W,Cin];
 * w: fp32 [Cout,Cin,ks,ks] (host); mode: 0 stride-1 pad ks/2, 1 stride-2 pad (1,1,1,1),
 * 2 stride-2 pad (0,1,0,1) (VAE encoder), 3 nearest-2x upsample then stride-1.  y: 16-bit NHWC.
 * GP_F16_PAIR through the implicit GEMM needs Cin % 8 == 0 (the lo plane of a pixel must start 16-byte aligned);
 * use_direct_kernel takes any Cin. */
gp_status gp_conv2d(int dtype, const void* x, int N, int H, int W, int Cin, const float* w_host,
                    const float* bias_host, int Cout, int ks, int mode, const void* residual, int relu,
                    void* y, int use_direct_kernel, void* stream);
gp_status gp_groupnorm(int dtype, const void* x, int N, int H, int W, int C, int groups, const float* gamma_host,
                       const float* beta_host, float eps, int silu, void* y, void* stream);
/* GroupNorm(groups, eps)(+SiLU) -> 3x3 stride-1 convolution (+ optional 1x1 shortcut over a RAW second tensor sc_x
 * [N,H,W,Csc], + optional residual): the norm1/conv1, norm2/conv2 (+conv_shortcut) and conv_norm_out/conv_out pairs of the
 * diffusers ResnetBlock2D / VAE heads, run as a GroupNorm pass, then the convolution.  y: 16-bit NHWC, or (out_f32 != 0)
 * fp32 NCHW [N,Cout,H,W]. */
gp_status gp_gn_conv3x3(int dtype, const void* x, int N, int H, int W, int Cin, int groups, const float* gamma_host,
                        const float* beta_host, float eps, int silu, const float* w_host, const float* bias_host, int Cout,
                        const void* sc_x, int Csc, const float* sc_w_host, const float* sc_b_host, const void* residual,
                        void* y, int out_f32, void* stream);
/* 3x3 stride-1 convolution x [N,H,W,Cin] -> y_conv [N,H,W,Cout] (16-bit NHWC, bias optional), then GroupNorm(groups,
 * eps)(+SiLU) over concat(y_conv, skip) -> y [N,H,W,Cout+Cskip]: the UNet up block's norm1 over [hidden | skip].  skip
 * (16-bit NHWC [N,H,W,Cskip]) may be NULL (Cskip = 0); a group may straddle the two sources.  In the 16-bit modes a
 * y_conv of Cout <= 512 (Cout % 64 == 0) carries its GroupNorm statistics out of the convolution's epilogue, as in the
 * engine; otherwise a statistics pass reads it.  Cout, Cskip: multiples of 8. */
gp_status gp_conv_groupnorm(int dtype, const void* x, int N, int H, int W, int Cin, const float* w_host, const float* bias_host,
                            int Cout, const void* skip, int Cskip, int groups, const float* gamma_host, const float* beta_host,
                            float eps, int silu, void* y_conv, void* y, void* stream);
gp_status gp_layernorm(int dtype, const void* x, int64_t tokens, int C, const float* gamma_host,
                       const float* beta_host, float eps, void* y, void* stream);
/* softmax(q k^T * scale) v per (batch, head); q,k,v,o: 16-bit [B,T,heads*d] */
gp_status gp_attention(int dtype, const void* q, const void* k, const void* v, int B, int T, int heads, int d,
                       float scale, void* o, void* stream);
/* replaces: the fp32 attention of the reference's default dtype, in the engine's high-precision layout (fp16 (hi, lo)
 * pairs, value = hi + lo).  softmax(q k^T) v per (batch, head), the softmax scale already folded into q as the engine folds
 * it into Wq.  qk: [B,T,4C] = per token [q hi | k hi | q lo | k lo] (C = heads * d each); v: [B,T,2C] = [v hi | v lo];
 * o: [B,T,2C] = [o hi | o lo].  d = 64 or (heads = 1) 512.  fused != 0: the fused split-precision kernel; 0: the unfused
 * QK^T -> softmax -> P V path (GP_ERR_INVALID where its softmax cannot take rows of T keys).  V^T goes through the
 * engine's own GEMM either way. */
gp_status gp_attention_high(const void* qk, const void* v, int B, int T, int heads, int d, int fused, void* o, void* stream);
/* replaces: the align / reduce / normalise tail of ensemble_depth (/root/reference/genpercept/util/ensemble.py:101-156,
 * 186-203): out[H,W] = median (torch.median: lower middle) or mean over the B <= 32 members of pred[b] * scale[b] + shift[b],
 * then (normalise 1) (x - min) / max(max - min, 1e-6) or (normalise 2) x / max(max, 1e-6).  pred / out: fp32 on the device. */
gp_status gp_ensemble_reduce(const float* pred_dev, int B, int H, int W, const float* scale_host, const float* shift_host,
                             int median, int normalise, float* out_dev, void* stream);
gp_status gp_bilinear_up2x(int dtype, const void* x, int N, int H, int W, int C, void* y, void* stream);
/* The UNet transformer's and up blocks' ops through the engine's own emission (the same ops, weights folding and packing
 * as a plan), each on caller buffers, synchronised.  dtype: GP_F16, GP_BF16 or GP_F16_PAIR; weights fp32 on the host, in
 * the checkpoint's layout.
 * gp_geglu: y [tokens,4C] = GEGLU(x [tokens,C] @ w^T + b), w [8C,C] and b [8C] as ff.net.0.proj stores them (values in rows
 * 0..4C-1, gates in 4C..8C-1; GELU with erf).  C % 8 == 0. */
gp_status gp_geglu(int dtype, const void* x, int64_t tokens, int C, const float* w_host, const float* b_host, void* y,
                   void* stream);
/* y [tokens,C] = x + attn2(LayerNorm(x; norm_g, norm_b, eps), ctx) with `heads` heads: to_q [C,C], to_k / to_v [C,E],
 * to_out [C,C] + [C], ctx [n,E] (host).  n = 2 takes the closed-form 2-token kernel (heads % 5 == 0, C <= 1280), any other n
 * the general path (LayerNorm, scores GEMM, per-head softmax, output GEMM).  C % 8 == 0, C % heads == 0. */
gp_status gp_cross_attention(int dtype, const void* x, int64_t tokens, int C, int heads, const float* ctx_host, int n, int E,
                             const float* to_q, const float* to_k, const float* to_v, const float* to_out_w,
                             const float* to_out_b, const float* norm_g, const float* norm_b, float eps, void* y,
                             void* stream);
/* ResnetBlock2D (32 groups, SiLU, no time embedding) over concat(x [N,H,W,Cx], skip [N,H,W,Cskip]) -> y [N,H,W,Cout]:
 * norm1 [Cin], conv1 [Cout,Cin,3,3] + [Cout], norm2 [Cout], conv2 [Cout,Cout,3,3] + [Cout], and the 1x1 conv_shortcut
 * [Cout,Cin,1,1] + [Cout], given exactly when Cin = Cx + Cskip != Cout (else the residual is x).  skip may be NULL
 * (Cskip = 0).  Channels: multiples of 8, Cin and Cout of 32. */
gp_status gp_resnet(int dtype, const void* x, int Cx, const void* skip, int Cskip, int N, int H, int W, int Cout, float eps,
                    const float* norm1_g, const float* norm1_b, const float* conv1_w, const float* conv1_b,
                    const float* norm2_g, const float* norm2_b, const float* conv2_w, const float* conv2_b,
                    const float* shortcut_w, const float* shortcut_b, void* y, void* stream);
/* F.interpolate(x [N,H,W,C], size=(OH,OW)) -> y [N,OH,OW,C]: mode 0 nearest (the UNet's Upsample2D to a skip's size),
 * 1 bilinear with align_corners=False (the DPT fusion stage's resize of a skip feature).  C % 8 == 0. */
gp_status gp_resize(int dtype, const void* x, int N, int H, int W, int C, int OH, int OW, int mode, void* y, void* stream);
/* The text tower's kernels (gp_encode_text), each on caller buffers, synchronised; dtype GP_F16, GP_BF16 or GP_F16_PAIR.
 * gp_causal_attention: out [n, C] = softmax(q k^T) v per head over keys j <= i (scores and softmax in fp32), C = heads * d,
 * from qkv [n, 3C] = per token [q | k | v] (the fused projection's output, the softmax scale already in q); pair layout:
 * per token [hi 3C | lo 3C] in, [hi C | lo C] out.  1 <= n <= 77, 1 <= d <= 64.
 * gp_gelu: y = x * (1 + erf(x / sqrt 2)) / 2 over n_elems values (n_elems % 8 == 0); pair layout: [hi n_elems | lo n_elems]. */
gp_status gp_causal_attention(int dtype, const void* qkv, int n, int heads, int d, void* out, void* stream);
gp_status gp_gelu(int dtype, const void* x, int64_t n_elems, void* y, void* stream);
/* ---- pre/post-processing around the hot path (SURVEY.md §8 f1); buffers may be host or device ------------
 * gp_resize_aa replaces torchvision.transforms.functional.resize(tensor, size, interpolation, antialias=True)
 * as called by resize_max_res (/root/reference/genpercept/util/image_util.py:75-105) and by the resize back
 * to the input resolution (/root/reference/genpercept/genpercept_pipeline.py:301-307): N planes [N,H,W] ->
 * [N,OH,OW]; src GP_U8 or GP_F32; dst GP_F32, or GP_U8 = round-half-even (+ clamp for bicubic) as torchvision
 * does for integer tensors; mode 0 bilinear, 1 bicubic.
 * The three pre/post entry points share one growing scratch buffer and the cached filter tables per device:
 * like gp_infer on one engine they are meant for one caller thread and stream-ordered use (calls on the same
 * stream, or separated by a synchronisation); they return after the copy whenever a host buffer is involved. */
gp_status gp_resize_aa(const void* src, int src_dtype, int src_on_host, int N, int H, int W, void* dst, int dst_dtype,
                       int dst_on_host, int OH, int OW, int mode, void* stream);
/* colorize_depth_maps + the uint8 cast at its call site (image_util.py:25-63, genpercept_pipeline.py:318-321):
 * pred f32 [B,H,W] -> u8 [B,H,W,3] = lut[clip(floor((x-vmin)/(vmax-vmin)*256), 0, 255)], lut = 256x3 u8 (host). */
gp_status gp_colorize(const float* pred, int pred_on_host, int B, int H, int W, float vmin, float vmax,
                      const uint8_t* lut768_host, uint8_t* out_hwc, int out_on_host, void* stream);
/* (pred*255).astype(uint8) / (pred*65535).astype(uint16) of /root/reference/run.py:449-455; bits = 8 or 16. */
gp_status gp_quantize(const float* pred, int pred_on_host, size_t n, int bits, void* out, int out_on_host, void* stream);
/* replaces: PIL.Image.Image.resize((OW, OH)) with its default filter (BICUBIC, reducing_gap=None) on a mode "RGB" image,
 * as GenPercept v1's resize_max_res / resize_res call it (GenPercept_v1/genpercept/util/image_util.py).  Byte-identical
 * to Pillow: the coefficient tables are Pillow's (double, normalised per window, 22-bit fixed point), built on the host
 * once per (in, out) extent and cached with gp_resize_aa's; the passes are integer only, the horizontal one over just the
 * rows the vertical one reads, and a pass whose extent is unchanged is skipped.  src: HWC uint8 [H,W,3] (Pillow's
 * storage order); dst: CHW uint8 [3,OH,OW], the layout gp_infer takes.  Buffers host or device, as gp_resize_aa. */
gp_status gp_resize_pil(const uint8_t* src_hwc, int src_on_host, int H, int W, uint8_t* dst_chw, int dst_on_host, int OH,
                        int OW, void* stream);
/* ---- baseline JPEG decoding (jpeg.cu); engine-free --------------------------------------------------------------
 * replaces: Image.open(path).convert("RGB") on a JPEG (run.py's input, decoded inside the reference's __call__):
 * RGB bytes identical to Pillow's (libjpeg-turbo, JDCT_ISLOW, fancy upsampling).  Taken: SOF0 / SOF1, 8-bit, three
 * components libjpeg infers as YCbCr (JFIF, Adobe transform 1, or ids 1-2-3), one interleaved scan, luma sampling
 * 1x1, 2x1 or 2x2 with 1x1 chroma, any restart interval.  Everything else is GP_ERR_INVALID.
 * gp_jpeg_probe is host only (no device needed): GP_OK with the frame size and the workspace the decode needs, or
 * GP_ERR_INVALID with the reason in gp_last_call_error().
 * gp_jpeg_decode uploads the file bytes into the caller's device workspace (>= the probed size; nothing is allocated),
 * decodes on `stream` and writes dst[y * row_stride + x * pixel_stride + c * channel_stride] (uint8, device; strides
 * in elements), then waits for the status word: GP_ERR_INVALID for a stream that is corrupt, whose markers are not
 * where they belong, or whose parallel Huffman decode did not converge (the caller decodes it another way). */
gp_status gp_jpeg_probe(const uint8_t* data, size_t nbytes, int* H, int* W, int64_t* workspace_bytes);
gp_status gp_jpeg_decode(const uint8_t* data_host, size_t nbytes, void* workspace_dev, int64_t workspace_bytes,
                         uint8_t* dst_dev, int64_t row_stride, int64_t pixel_stride, int64_t channel_stride,
                         void* stream);
/* replaces: the post-processing of GenPercept v1's __call__ (GenPercept_v1/genpercept/pipeline_genpercept.py) on the
 * engine's map.  pred: fp32 [B,C,h,w] in [0,1] on the device (gp_infer's out); p = 2 pred - 1 is v1's single_infer result.
 * p is taken to (H, W) by F.interpolate (task 0 / 1: bilinear, align_corners=False, no antialiasing; task 2: the legacy
 * nearest), skipped when (H, W) == (h, w).  Then, all device buffers:
 *   task 0 depth (C = 1):  out_f32 [B,H,W] = (x - min) / (max - min) per image, unclamped (a constant map gives NaN);
 *                          the min / max come from per-block partials reduced in a fixed order
 *   task 1 normal (C = 3): out_f32 [B,3,H,W] = clip(x, -1, 1); out_u8 [B,H,W,3] = norm_to_rgb of it (float32 arithmetic)
 *   task 2 seg / sr (C = 3): out_u8 [B,3,H,W] = ((x + 1) / 2 * 255).clip(0, 255).astype(uint8)
 * Asynchronous on `stream`; shares the pre/post scratch above. */
gp_status gp_v1_postprocess(const float* pred, int B, int C, int h, int w, int task, int H, int W, float* out_f32,
                            uint8_t* out_u8, void* stream);
/* ---- depth evaluation (SURVEY.md §8 f4): the reference's eval.py loop on the device; engine-free ------------------
 * pred, gt: fp32 [B,H,W]; valid: uint8 [B,H,W] (nonzero = valid; NULL = every pixel); all device pointers.  Both
 * calls use the pre/post scratch buffer above, return asynchronously on `stream`, and are bit-identical run to run.
 * gp_depth_align replaces align_depth_least_square (/root/reference/src/util/alignment.py:29-76): per image the
 * (scale, shift) np.linalg.lstsq fits to gt over the valid pixels, rounded to float32 -> scale_shift_out [B,2] (device).
 * mode 0 fits gt as given; 1 the disparity mode of eval.py:177-197 (target 1/gt where gt > 0, mask valid & gt > 0 &
 * pred > 0).  max_res > 0: the fit reads the grid torch.nn.Upsample(scale_factor=min(max_res/(H,W)), "nearest") makes
 * of the [1,H,W] map when that factor is below 1 (a 1-D resample: H x floor(W*s)); 0 = none.  No pixel valid -> (0, 0);
 * a constant prediction -> lstsq's minimum-norm solution.  aligned_out (nullable): fp32 [B,H,W] pred*scale + shift. */
gp_status gp_depth_align(const float* pred, const float* gt, const uint8_t* valid, int B, int H, int W, int mode,
                         int max_res, float* scale_shift_out, float* aligned_out, void* stream);
/* The ten metrics of eval.py:42-53 per image -> metrics_out fp64 [B,10] (device), in that order: abs_relative_difference,
 * squared_relative_difference, rmse_linear, rmse_log, log10, delta1_acc, delta2_acc, delta3_acc, i_rmse, silog_rmse.
 * Per pixel (float32, eval.py:168-205): mode 0 pred as given; 1 pred*scale+shift; 2 the same, clipped at 1e-3 and
 * inverted (disparity -> depth); then clip to [min_depth, max_depth] and to >= 1e-6.  scale_shift: [B,2] on the device
 * (gp_depth_align's output; unused in mode 0).  No pixel valid -> NaN metrics, like the reference. */
gp_status gp_depth_metrics(const float* pred, const float* gt, const uint8_t* valid, int B, int H, int W, int mode,
                           const float* scale_shift, float min_depth, float max_depth, double* metrics_out, void* stream);

/* time one igemm configuration: returns average microseconds over `iters` launches */
gp_status gp_bench_conv(int dtype, int N, int H, int W, int Cin, int Cout, int ks, int mode, int iters,
                        double* usec, double* flops);
/* time one path of the single-head d = 512 attention (the VAE mid-block) on B images of T tokens: fused != 0 the fused
 * kernel, 0 the unfused QK^T -> softmax -> P V path, whichever the planner would pick for that size.  Returns the
 * average microseconds over `iters` calls after one warm-up call, and the algorithmic FLOPs (4 B T^2 512) of one call. */
gp_status gp_bench_attention(int dtype, int B, int T, int fused, int iters, double* usec, double* flops);
/* time one path of the high-precision attention (as gp_attention_high) on B images of T tokens, `heads` heads of d = 64
 * or one of d = 512: fused != 0 the fused split-precision kernel, 0 the unfused path (GP_ERR_INVALID where it cannot run).
 * Returns the average microseconds over `iters` calls after one warm-up call, and the algorithmic FLOPs (4 B heads T^2 d). */
gp_status gp_bench_attention_high(int B, int T, int heads, int d, int fused, int iters, double* usec, double* flops);

#ifdef __cplusplus
}
#endif
#endif
