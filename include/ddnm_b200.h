/* ddnm_b200 — C ABI of the H100-native DDNM sampling engine (libddnm_b200.so).
 *
 * The reference (wyhuai/DDNM) has no FFI: its hot path is reached through three Python call conventions
 * (SURVEY.md §8b).  Each entry point below names the reference interface it stands behind; the Python
 * shims in ddnm_b200/{model,operators,sampler}.py keep those signatures and forward to these symbols
 * via ctypes (INTEGRATION.md shows the binding).
 *
 * Conventions: every pointer is a raw CUDA device pointer unless a comment says "host"; `stream` is a
 * cudaStream_t (NULL = default stream); work is enqueued asynchronously on it; tensors are borrowed
 * for the duration of the call, workspaces belong to the handle.  Return value 0 = ok, non-zero =
 * failure with a message available from ddnm_last_error() (thread-local).  Handles are per device and
 * not re-entrant.
 */
#ifndef DDNM_B200_H
#define DDNM_B200_H

#ifdef __cplusplus
extern "C" {
#endif

const char* ddnm_last_error(void);
int ddnm_version(void);

/* ------------------------------------------------------------------------------------------------
 * Denoiser: guided_diffusion/models.py::Model ("simple" DDPM UNet of configs/celeba_hq.yml).
 * Replaces `et = model(xt, t)` at functions/svd_ddnm.py:47,108 (Model.forward, models.py:301-341).
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  int ch, out_ch, n_levels;
  int ch_mult[8];
  int num_res_blocks;
  int n_attn_res;
  int attn_res[4];
  int in_channels, resolution, groups;
  float eps;
} ddnm_simple_cfg;   /* mirrors config.model.* / config.data.image_size read at models.py:195-204 */

int ddnm_unet_simple_create(const ddnm_simple_cfg* cfg, int batch, void** handle);

/* Denoiser: guided_diffusion/unet.py::UNetModel as built by script_util.create_model (:130-185) for imagenet_256.yml:
 * use_scale_shift_norm, resblock_updown, legacy attention order, class_cond = false.  Replaces `et = model(xt, t)` for
 * model.type == "openai" (UNetModel.forward, unet.py:635-664).  Parameter names = UNetModel.state_dict() keys
 * (Conv1d qkv / proj_out weights keep their (O, I, 1) layout); "__freq" = exp(-log(1e4) * arange(mc/2) / (mc/2))
 * (nn.py:113-115).  All handle functions below (set_param ... destroy) accept either denoiser kind. */
typedef struct {
  int image_size, model_channels, num_res_blocks, n_levels;
  int channel_mult[8];
  int n_attn_ds;
  int attn_ds[4];             /* image_size // attention resolution, as create_model computes (:163-165) */
  int num_head_channels, out_channels, in_channels, groups;
  float eps;
  int num_classes;            /* 0 = unconditional; > 0 = class_cond (imagenet_256_cc.yml): label_emb.weight [num_classes, 4*ch],
                                 emb = time_embed(t) + label_emb(y) (unet.py:478-479, 651-653) */
} ddnm_openai_cfg;
int ddnm_unet_openai_create(const ddnm_openai_cfg* cfg, int batch, void** handle);
/* name = key of Model.state_dict() (models.py:216-299), data = fp32 host or device, reference layout (OIHW);
 * plus the pseudo-parameter "__freq" = exp(arange(ch/2) * -log(1e4)/(ch/2-1)) (models.py:16-18). */
int ddnm_unet_set_param(void* handle, const char* name, const float* data, long long numel);
/* Arithmetic of the tensor-core contractions, to be chosen before finalize: 3 (default) = every fp32 product as
 * hi*hi + hi*lo + lo*hi of fp16 pairs (fp32-grade, the parity mode); 1 = one fp16 product per MAC with fp32 accumulation
 * (fast mode; comparable to the reference's own use_fp16 torso, unet.py:619-625, NOT within rtol 1e-3 of the fp32 model). */
int ddnm_unet_set_precision(void* handle, int fp16_terms);
int ddnm_unet_finalize(void* handle);
/* x [B,3,R,R] NCHW fp32, t [B] fp32 holding integer timesteps, out [B,out_ch,R,R] NCHW fp32 */
int ddnm_unet_forward(void* handle, const float* x, const float* t, float* out, void* stream);
/* class-conditional networks: `model(x, t, y)` (UNetModel.forward(x, timesteps, y), unet.py:635-653); labels = device int32 [B] */
int ddnm_unet_forward_cond(void* handle, const float* x, const float* t, const int* labels, float* out, void* stream);
int ddnm_unet_set_graph(void* handle, int use_cuda_graph);
int ddnm_unet_read_tap(void* handle, const char* name, float* dst_nchw, long long capacity, void* stream);
int ddnm_unet_info(void* handle, long long* workspace_bytes, int* launches, double* flops_per_forward);
/* per-launch CUDA-event timing of one eager forward, JSON array into json (host) */
int ddnm_unet_profile(void* handle, const float* x, const float* t, float* out, void* stream, char* json, long long capacity);
int ddnm_unet_destroy(void* handle);

/* ------------------------------------------------------------------------------------------------
 * Degradation operators: functions/svd_operators.py A_functions contract (:52-97):
 * A, A_pinv, Lambda, Lambda_noise, plus the fused projection x0 - A^+(A x0 - y) of svd_ddnm.py:59-61.
 * kind: 0 SuperResolution(:479) 1 Colorization(:627) 2 Inpainting(:324) 3 WalshHadamardCS(:211)
 *       4 Deblurring(:934) 5 SRConv(:851) 6 Denoising(:442) 7 Deblurring2D(:1094) 8 CS(:101; `ratio` = cs_size,
 *       v_small = the 1024x1024 basis)  9 GeneralA(:173; dense A = U diag(s) V^T: `ratio` = m rows of A,
 *       v_small = V [n,n] with n = channels*img_dim^2, u_small = U [m,m], singulars [m] already thresholded; no Lambda).
 * Artefacts (V_small, perm, mask, singular tables) are inputs.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  int kind, channels, img_dim, ratio;
  const float* v_small;       /* SR: [r*r, r*r]; Colorization: [3,3]; Deblurring/SRConv: V_small [dim,dim] */
  const float* u_small;       /* SR/Colorization: [1,1]; Deblurring: [dim,dim]; SRConv: [small,small] */
  const float* singulars;     /* SR/Colorization: [1]; Deblurring: sorted big singulars [dim*dim]; SRConv: small [small] */
  const float* singulars_orig;/* Deblurring: un-thresholded, sorted [dim*dim] */
  const long long* perm;      /* WalshHadamardCS: [dim*dim]; Deblurring: [dim*dim] */
  const long long* mask;      /* Inpainting: [dim*dim*channels] keep flags over the (pixel, channel)-interleaved vector the
                                 reference's missing_indices address (diffusion.py:466-470); 0 = missing */
  const float* v_small2;      /* Deblurring2D: V_small2 [dim,dim] (right-hand factor); others NULL */
  const float* u_small2;      /* Deblurring2D: U_small2 [dim,dim] */
} ddnm_operator_desc;         /* all pointers: host memory, copied at creation */

int ddnm_operator_create(const ddnm_operator_desc* desc, void** handle);
long long ddnm_operator_y_dim(void* handle);                       /* M = length of A(x) per image */
int ddnm_operator_A(void* handle, const float* x, int B, float* y, void* stream);
int ddnm_operator_A_pinv(void* handle, const float* y, int B, float* x, void* stream);
int ddnm_operator_project(void* handle, const float* x0, const float* y, int B, float* x0_hat, void* stream);
/* Lambda / Lambda_noise (svd_operators.py:91-97 and per class, coefficient rule e.g. :568-604); a = sqrt(alpha-bar_next),
 * sigma_t = sqrt(1 - alpha-bar_next) as fp32 scalars, sigma_y and eta as the reference's python floats */
int ddnm_operator_lambda(void* handle, const float* v, int B, float a, float sigma_y, float sigma_t, float eta, float* out,
                         void* stream);
int ddnm_operator_lambda_noise(void* handle, const float* v, const float* eps, int B, float a, float sigma_y, float sigma_t,
                               float eta, float* out, void* stream);
int ddnm_operator_destroy(void* handle);

/* ------------------------------------------------------------------------------------------------
 * Sampler: functions/svd_ddnm.py ddnm_diffusion (:19-78) / ddnm_plus_diffusion (:80-164).
 * One fused kernel per time pair does x0_t, the null-space projection (and Lambda / Lambda_noise for DDNM+)
 * and the re-noising; the whole loop is enqueued without host synchronisation.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  int n_pairs;
  const int* t_i;             /* host [n_pairs]: model time of the pair's source */
  const int* t_j;             /* host [n_pairs]: target time (-1 = final) ; j > i = travel-back step */
  const float* abar;          /* host [num_timesteps+1]: cumprod table, abar[t+1] = alpha-bar(t), abar[0] = 1 */
  int num_timesteps;
  float eta;
  float sigma_y;              /* DDNM+: measurement noise level (already doubled, diffusion.py:524) */
  int plus;                   /* 0 = ddnm_diffusion update (:57-65), 1 = ddnm_plus_diffusion update (:114-131) */
} ddnm_schedule;

/* x_T [B,3,R,R]; y [B,M]; noise [n_pairs,B,3,R,R] (the randn_like draws of svd_ddnm.py:65,74 in order);
 * out_x0 [B,3,R,R] = xs[-1]; out_x0_pred [B,3,R,R] = x0_preds[-1] (may be NULL). */
int ddnm_sample(void* unet, void* op, const ddnm_schedule* sched, const float* x_T, const float* y, const float* noise, int B,
                float* out_x0, float* out_x0_pred, void* stream);

/* Class-conditional / classifier-guided sampling (svd_ddnm.py:48-52, :109-113; imagenet_256_cc.yml):
 *   et = model(xt, t, classes)[:, :3];  et = et - sqrt(1 - at) * cls_fn(x, t, classes)
 * labels: device int32 [B] handed to the class-conditional denoiser (NULL for an unconditional one).
 * fn (may be NULL): called on the calling thread once per denoising pair, after the denoiser was enqueued; it must leave
 * cls_fn's result in grad_buf (device [B,3,R,R]) using work enqueued on `stream` and return 0.  The classifier and its
 * backward pass stay with the caller (the reference builds them from PyTorch autograd, diffusion.py:181-189). */
typedef int (*ddnm_guidance_fn)(void* user, int pair_index, int t, void* stream);
int ddnm_sample_guided(void* unet, void* op, const ddnm_schedule* sched, const float* x_T, const float* y, const float* noise, int B,
                       const int* labels, const float* grad_buf, ddnm_guidance_fn fn, void* user, float* out_x0, float* out_x0_pred,
                       void* stream);

/* Bounded-memory form of the same loop: pairs [k_begin, k_end) of the schedule, state in the caller's buffers, so a long
 * schedule (T_sampling = 1000, time-travel) runs as several calls that each see only their own slice of the noise draws
 * (the reference needs O(1) noise memory: one torch.randn_like per pair, svd_ddnm.py:65,74).
 *   xt       [B,3,R,R] in/out: the iterate (x_T before the first range, xs[-1] after the last)
 *   x0_pred  [B,3,R,R] in/out: the last UN-projected x0_t (travel-back pairs read it); *have_x0 (host int, in/out) says whether
 *            it holds one yet (0 before the first range)
 *   noise    [(k_end - k_begin),B,3,R,R]: the draws of exactly these pairs
 * labels / grad_buf / fn / user as in ddnm_sample_guided (all NULL for the unguided loop). */
int ddnm_sample_range(void* unet, void* op, const ddnm_schedule* sched, int k_begin, int k_end, float* xt, float* x0_pred,
                      int* have_x0, const float* y, const float* noise, int B, const int* labels, const float* grad_buf,
                      ddnm_guidance_fn fn, void* user, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Classifier of guided sampling: guided_diffusion/unet.py::EncoderUNetModel (unet.py:684-895) as create_classifier builds it
 * for imagenet_256_cc.yml (use_scale_shift_norm, resblock_updown, legacy attention, 64-channel heads).  Parameters go through
 * ddnm_unet_set_param / set_precision / finalize / set_graph / info / profile / destroy with EncoderUNetModel.state_dict() keys
 * (Conv1d weights keep their (O, I, 1) data) plus "__freq" (the timestep-embedding frequencies).
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  int image_size, model_channels, num_res_blocks, n_levels;
  int channel_mult[8];
  int n_attn_ds;
  int attn_ds[4];             /* downsample rates at which attention runs */
  int num_head_channels, out_channels, in_channels, groups;
  float eps;
  int pool;                   /* 0 = "adaptive", 1 = "attention" */
} ddnm_classifier_cfg;
int ddnm_classifier_create(const ddnm_classifier_cfg* cfg, int batch, void** handle);
/* x [B,3,R,R], t [B] fp32 (device) -> logits [B, out_channels] */
int ddnm_classifier_forward(void* h, const float* x, const float* t, float* logits, void* stream);
/* grad_out [B,3,R,R] = scale * d/dx sum_b log_softmax(classifier(x, t))[b, labels[b]]  (cond_fn, diffusion.py:183-189);
 * labels: device int32 [B], each in [0, out_channels) (checked: the call synchronises `stream` to read them);
 * logits_out [B, out_channels] may be NULL.  No parameter gradients. */
int ddnm_classifier_grad(void* h, const float* x, const float* t, const int* labels, float scale, float* grad_out, float* logits_out,
                         void* stream);
/* Native classifier guidance for ddnm_sample_guided / ddnm_sample_range: pass ddnm_classifier_guidance_fn as `fn` and a
 * ddnm_classifier_guidance as `user`; each call leaves the gradient at (x, t) in grad_buf (the loop's grad_buf), with work enqueued on
 * the loop's stream and no host synchronisation after the first call. */
typedef struct {
  void* classifier;           /* ddnm_classifier_create handle built for the sampler's batch */
  const float* x;             /* device [B,3,R,R]: where the gradient is taken */
  const int* labels;          /* device int32 [B] */
  float scale;
  float* grad_buf;            /* device [B,3,R,R] */
  int batch;                  /* B of the guided loop: must equal the classifier's batch */
  int labels_checked;         /* 0 before the loop; set to 1 once the labels were range-checked (then never re-read to the host) */
} ddnm_classifier_guidance;
int ddnm_classifier_guidance_fn(void* user, int pair_index, int t, void* stream);

/* ------------------------------------------------------------------------------------------------
 * "Simplified" DDNM+ (guided_diffusion/diffusion.py:211-415, the README quick-start path): image-space operators composed
 * of mask (A1 = z*mask, :256), colour->gray (color2gray/gray2color, :33-42) and average pooling (AdaptiveAvgPool2d /
 * MeanUpsample, :27-31,:252-253), with the scalar lambda_t / gamma_t update of :355-381.  deg table (:244-290):
 *   colorization = gray; denoising = none; sr_averagepooling = scale; inpainting = mask; mask_color_sr / diy = all three.
 * y and A's output are (B, 3, D/scale, D/scale) fp32 (gray replicates its value over the 3 channels, as the reference).
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  int use_mask, use_gray, scale, img_dim, channels;
  const float* mask;          /* DEVICE [img_dim*img_dim] 0/1 (exp/inp_masks/mask.npy), NULL when use_mask == 0 */
} ddnm_simple_deg;
int ddnm_simplified_A(const ddnm_simple_deg* deg, const float* x, int B, float* y, void* stream);
int ddnm_simplified_Ap(const ddnm_simple_deg* deg, const float* y, int B, float* x, void* stream);
/* schedule->sigma_y is the doubled level (diffusion.py:292); schedule->plus is ignored */
int ddnm_sample_simplified(void* unet, const ddnm_simple_deg* deg, const ddnm_schedule* sched, const float* x_T, const float* y,
                           const float* noise, int B, float* out_x0, float* out_x0_pred, void* stream);

/* pairs [k_begin, k_end) with caller-held state: same contract as ddnm_sample_range */
int ddnm_sample_simplified_range(void* unet, const ddnm_simple_deg* deg, const ddnm_schedule* sched, int k_begin, int k_end, float* xt,
                                 float* x0_pred, int* have_x0, const float* y, const float* noise, int B, void* stream);

/* ------------------------------------------------------------------------------------------------
 * hq_demo: arbitrary-size restoration with the mask-shift trick (hq_demo/guided_diffusion/gaussian_diffusion.py:318-390 "DDNM core",
 * :431-493 p_sample, :208-217 _undo, :578-750 window loop).  The window / time loops are host code (ddnm_b200/hq.py, as in the
 * reference); these entry points do the tensor work of one step on 256 x 256 windows.
 *   ddnm_hq_canvas: Apy_temp = Ap(A_temp(gt)) for gt (B,3,H,W), H % scale == W % scale == 0 (:651-655; use_gray: colour->gray first)
 *   ddnm_hq_step  : x0_t = clip(c_recip*x - c_recipm1*eps); x0_hat = lambda_t*Apy + x0_t - lambda_t*Ap(A(x0_t)); the two
 *                   rectangles rects[0..5], rects[6..11] = {dst_y, dst_x, h, w, src_y, src_x} (h == 0: unused) of x0_hat are
 *                   overwritten from the canvas (:344-384); mean = coef1*x0_hat + coef2*x (+ gamma_t*grad, :414-430);
 *                   x_next = mean + nonzero*sqrt(gamma_t)*noise.  scratch: 3*B*3*D*D floats.
 *   ddnm_hq_undo  : x = sqrt(1-beta)*x + sqrt(beta)*noise (time-travel back step)
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  float c_recip, c_recipm1;   /* sqrt_recip_alphas_cumprod[t], sqrt_recipm1_alphas_cumprod[t] */
  float coef1, coef2;         /* posterior_mean_coef1[t], posterior_mean_coef2[t] */
  float lambda_t, gamma_t;    /* Eq. 19 */
  float nonzero;              /* 0 at t == 0, else 1 */
  int clip;                   /* clip_denoised */
} ddnm_hq_scalars;
int ddnm_hq_canvas(const float* gt, int B, int H, int W, int scale, int use_gray, float* apy_canvas, void* stream);
int ddnm_hq_step(const ddnm_simple_deg* deg, const float* x, const float* model_out, int out_ch, const float* apy, const float* canvas,
                 int canvas_h, int canvas_w, const int* rects, const float* grad, const float* noise, const ddnm_hq_scalars* sc, int B,
                 float* x0_hat, float* x_next, float* scratch, void* stream);
int ddnm_hq_undo(float* x, const float* noise, float sqrt_one_minus_beta, float sqrt_beta, long long n, void* stream);

/* ------------------------------------------------------------------------------------------------
 * The runner's I/O step either side of the loop (guided_diffusion/diffusion.py:533-603), device pointers throughout.
 * ddnm_data_transform         = datasets/__init__.py:201-213 data_transform.  uniform_noise / gauss_noise: the torch.rand_like /
 *                               torch.randn_like draws of config.data.{uniform,gaussian}_dequantization, NULL when the flag is off;
 *                               rescaled / logit = config.data.rescaled / logit_transform (rescaled wins, as in the reference).
 * ddnm_inverse_data_transform = datasets/__init__.py:216-227 (sigmoid | (x+1)/2, clamp to [0,1]).
 * (`config.image_mean` is set by no shipped config; the Python shim rejects it.)
 * ddnm_finish_images: one pass over the restored batch x [B,C,H,W] (model space):
 *   out01      [B,C,H,W] fp32 = inverse_data_transform(x)                                    (NULL to skip)
 *   out_u8_hwc [B,H,W,C] uint8 = the bytes torchvision.utils.save_image encodes,
 *              mul(255).add_(0.5).clamp_(0,255).to(uint8)  (diffusion.py:596-598)              (NULL to skip)
 *   psnr       [B] = 10*log10(1 / mean((out01 - inverse_data_transform(orig))^2))  (diffusion.py:599-601); orig, psnr both NULL to skip
 * ---------------------------------------------------------------------------------------------- */
int ddnm_data_transform(const float* x, long long n, const float* uniform_noise, const float* gauss_noise, int rescaled, int logit,
                        float* out, void* stream);
int ddnm_inverse_data_transform(const float* x, long long n, int rescaled, int logit, float* out, void* stream);
int ddnm_finish_images(const float* x, const float* orig, int B, int C, int H, int W, int rescaled, int logit, float* out01,
                       unsigned char* out_u8_hwc, float* psnr, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Op-level entry points (unit tests, micro-benchmarks).  NHWC fp32 tensors, OIHW weights.
 * mode: 0 = 3x3 pad 1, 1 = 1x1, 2 = 3x3 stride 2 pad (0,1,0,1); up2: nearest x2 before the conv.
 * ---------------------------------------------------------------------------------------------- */
int ddnm_conv_tc(const float* x, int N, int H, int W, int Cin, const float* w, const float* bias, int Cout, int mode, int up2,
                 const float* side_x, int CinSide, const float* side_w, const float* residual, float* out, void* stream);
int ddnm_conv_direct(const float* x, int N, int H, int W, int Cin, const float* w, const float* bias, int Cout, int mode, int up2,
                     float* out, void* stream);
/* iters > 0: all-zero operands; iters < 0: |iters| iterations on pseudo-random operands (power-realistic) */
int ddnm_conv_tc_bench(int N, int H, int W, int Cin, int Cout, int mode, int iters, float* ms_per_iter, double* flops);
/* diag probe: GroupNorm+SiLU+split -> 3x3 convolution over N images in chunks of `chunk` images sharing one chunk-sized plane scratch */
int ddnm_gnconv_chunk_bench(int N, int chunk, int H, int W, int Cin, int Cout, int iters, float* ms_per_pass);
int ddnm_groupnorm(const float* x, int N, int H, int W, int C, int groups, const float* gamma, const float* beta, float eps,
                   int silu, float* out, void* stream);
/* out = conv3x3(silu?(groupnorm(x))) [+ conv1x1(side_x)] + bias [+ residual] with the GroupNorm / SiLU / fp16 split applied INSIDE the
 * convolution kernel (models.py:115-134 conv1 / conv2 + nin_shortcut), rows of >= 128 pixels.  gamma == NULL: no normalisation.
 * iters > 0 additionally times `iters` launches into *ms_per_iter. */
int ddnm_conv_gn_tc(const float* x, int N, int H, int W, int Cin, int groups, const float* gamma, const float* beta, float eps, int silu,
                    const float* w, const float* bias, int Cout, const float* side_x, int CinSide, const float* side_w,
                    const float* residual, float* out, int iters, float* ms_per_iter, void* stream);
/* 1: eligible layers (3x3, rows >= 128 pixels) of engines built afterwards run the fused GroupNorm convolution; 0 (default, also env
 * DDNM_GN_FUSED): gn_apply_kernel + conv_tc_kernel */
int ddnm_tc_debug_gn_fused(int on);
/* tuning experiments: force the N-tile width (64 or 128) of conv launches built afterwards (0 = heuristic) */
int ddnm_tc_debug_force_bn(int bn);
/* tile -> CTA map of conv launches built afterwards: -1 (default) contiguous tile ranges per CTA on layers with one N tile that
 * produce GroupNorm sums, 0 round-robin everywhere, 1 contiguous wherever legal */
int ddnm_tc_debug_deal(int mode);
/* CTA pairs (cluster of 2 sharing the weight tile through TMA multicast) for conv launches built afterwards: -1 (default) and 0
 * never (slower than single CTAs on the H100 networks), 1 wherever legal */
int ddnm_tc_debug_pair_mode(int mode);
/* 1 (default): single-CTA launches issue hi*hi and hi*lo as one m64 x 2BN instruction (two partial accumulators); 0: never */
int ddnm_tc_debug_dual_mode(int mode);
/* 1 (default): CTA pairs use that DUAL form as well; 0: the plain three-instruction pair form */
int ddnm_tc_debug_pair_dual(int on);
/* 1 (default, also env DDNM_HALO): 3x3 stride-1 and upsample-phase conv launches built afterwards on maps >= 64 px wide and without
 * a 1x1 side input load each
 * (dy, 64-channel slice) of the activation once as halo rows for all column taps; 0: one A load per tap */
int ddnm_tc_debug_halo(int on);
/* 1 (default, also env DDNM_PINGPONG): single-CTA launches without the fused GroupNorm form, built afterwards, run on the ping-pong
 * kernel (two consumer warpgroups that each own a whole tile and take turns on the tensor cores) where a CTA gets at least two tiles;
 * 0: never */
int ddnm_tc_debug_pingpong(int on);

#ifdef __cplusplus
}
#endif
#endif /* DDNM_B200_H */
