/* dip.h -- C ABI of libdip.so, the H100-native deep-image-prior hot-path engine.
 *
 * The reference (DmitryUlyanov/deep-image-prior) has no FFI: its hot path sits behind plain Python call sites.
 * Every entry point below names the reference call site it replaces (file:line into the reference repo).
 * The Python side (deep-image-prior_b200/dip_engine.py, ctypes) binds exactly these symbols; see INTEGRATION.md.
 *
 * Conventions: all device buffers are caller-owned (the Python side allocates them with torch so that autograd,
 * state_dict and the caching allocator keep working); calls are asynchronous on the given stream and never
 * synchronise; nothing throws across the ABI: 0 = success, negative = error, text via dip_last_error().
 * Activations inside the engine are fp32 NHWC; tensors crossing the ABI are torch-layout (NCHW / OIHW) fp32.
 */
#ifndef DIP_H_
#define DIP_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct dip_plan dip_plan;
typedef struct dip_adam dip_adam;
typedef void* dip_stream_t; /* cudaStream_t */

enum { DIP_PRECISION_TF32 = 0, /* wgmma tf32 convolutions, fp32 accumulate (cuDNN's default fp32 mode) */
       DIP_PRECISION_FP32 = 1, /* exact-fp32 CUDA-core convolutions (parity mode) */
       DIP_PRECISION_BF16 = 2  /* wgmma bf16 convolutions on bf16 operands (activations, gradients and weights rounded
                                  to bf16 where a convolution reads them), fp32 accumulate; fp32 master weights, BatchNorm,
                                  loss and Adam (BASELINE.json configs[2]: "super-resolution ... bf16") */ };

/* Arguments of models.skip(...) that the engine supports (reference: models/skip.py:5-11, models/__init__.py:12-17). */
typedef struct {
  int in_channels;       /* num_input_channels, 1..128 (32 in every BASELINE config; 3 in flash-no-flash)  */
  int out_channels;      /* num_output_channels (<= 4; 3)                                               */
  int num_scales;        /* len(num_channels_down)                                                      */
  int channels;          /* num_channels_down[i] == num_channels_up[i] (128 in every BASELINE configuration);
                            0: per-scale widths in channels_down / channels_up / channels_skip below     */
  int skip_channels;     /* num_channels_skip[i]: 0, 4, or 128 (inpainting.ipynb kate; 128-wide networks only) */
  int upsample_bilinear; /* upsample_mode: 1 'bilinear', 0 'nearest', -1: per scale, see upsample_mask  */
  int need_sigmoid;      /* 1: nn.Sigmoid behind the head (models/skip.py:97-98), 0: none                */
  int precision;         /* DIP_PRECISION_*                                                             */
  int upsample_mask;     /* upsample_bilinear == -1: bit i set = scale i (0 = outermost) is 'bilinear'
                            (flash-no-flash.ipynb c8: ['nearest','nearest','bilinear','bilinear','bilinear']) */
  int input_grad;        /* 1: dip_backward also prepares dL/d(net_input) for dip_input_grad
                            (OPT_OVER = 'net,input', utils/common_utils.py:47-49); costs two extra level-0 launches */
  /* channels == 0: widths per scale (index 0 = outermost), multiples of 8 in [8, 128]; skips 0 or 4 per scale
     (denoising.ipynb c8:17-23 "snail": down = up = [8, 16, 32, 64, 128], skip = [0, 0, 0, 4, 4])           */
  int channels_down[8];  /* num_channels_down (models/skip.py:6)                                        */
  int channels_up[8];    /* num_channels_up   (models/skip.py:6)                                        */
  int channels_skip[8];  /* num_channels_skip (models/skip.py:7)                                        */
  int downsample_mode;   /* 0: 'stride' (stride-2 conv); 1: 'avg' (stride-1 conv + AvgPool2d(2, 2), models/common.py:101-105,
                            restoration.ipynb c7:28-36 kate)                                            */
} dip_net_desc;

const char* dip_last_error(void);
int dip_version(void);

/* ---- plan: shapes -> buffers, TMA tensor maps, kernel schedule (replaces nn.Sequential.__call__ over the module
 *      tree built by models/skip.py:41-100).  Parameter order = net.parameters() order of the reference
 *      (depth-first: skip conv/bn, down conv/bn x2, <deeper level>, concat bn, up conv/bn, 1x1 conv/bn; head last). */
size_t dip_plan_workspace_bytes(const dip_net_desc* desc, int H, int W);
int dip_plan_create(const dip_net_desc* desc, int H, int W, void* workspace, size_t workspace_bytes,
                    dip_plan** out);

/* Plan options beyond dip_net_desc: the struct is {pad_mode, act_fun}, and a zero-initialised one (or opts == NULL) is
 * reflection padding with LeakyReLU.
 * pad_mode = the `pad` argument of models.skip (reference: models/common.py:114-120): DIP_PAD_REFLECTION inserts
 * nn.ReflectionPad2d before every 3x3 conv; any other value of `pad` gives Conv2d(padding=1), i.e. DIP_PAD_ZERO.
 * act_fun = the `act_fun` string of models.skip (reference: models/common.py:76-92), the activation behind every
 * BatchNorm except the concat's: 'LeakyReLU' = nn.LeakyReLU(0.2), 'Swish' = x * sigmoid(x), 'ELU' = nn.ELU() (alpha 1),
 * 'none' = the identity.
 * Every combination needs the same workspace.  Other values are rejected (dip_last_error() names the field). */
enum { DIP_PAD_REFLECTION = 0, DIP_PAD_ZERO = 1 };
enum { DIP_ACT_LEAKY_RELU = 0, DIP_ACT_SWISH = 1, DIP_ACT_ELU = 2, DIP_ACT_NONE = 3 };
typedef struct {
  int pad_mode;          /* DIP_PAD_*                                                                     */
  int act_fun;           /* DIP_ACT_*                                                                     */
} dip_plan_opts;
/* as dip_plan_workspace_bytes / dip_plan_create; opts may be NULL (= reflection padding and LeakyReLU, what the two calls
 * above use) */
size_t dip_plan_workspace_bytes_opts(const dip_net_desc* desc, int H, int W, const dip_plan_opts* opts);
int dip_plan_create_opts(const dip_net_desc* desc, int H, int W, const dip_plan_opts* opts, void* workspace,
                         size_t workspace_bytes, dip_plan** out);
void dip_plan_destroy(dip_plan* plan);
int dip_plan_num_params(const dip_plan* plan);
int dip_plan_num_bn(const dip_plan* plan);
long long dip_plan_param_numel(const dip_plan* plan, int index);
/* params[i], grads[i]: fp32 device buffers in torch layout; bn_running: 3 pointers per BatchNorm
 * (running_mean, running_var, num_batches_tracked) or NULL; nbt_is_float = 1 when num_batches_tracked is float32
 * (after Module.type(torch.cuda.FloatTensor)), 0 for torch's native int64.  May be called again when pointers change. */
int dip_plan_bind(dip_plan* plan, void* const* params, void* const* grads, void* const* bn_running,
                  int nbt_is_float);

/* out = net(z + sigma * noise)      (reference: `out = net(net_input)`, denoising.ipynb c10:12-15)
 * z, noise: [C_in][H][W] fp32 (noise may be NULL); out: [C_out][H][W].  Training-mode BatchNorm statistics. */
int dip_forward(dip_plan* plan, const void* z, const void* noise, float sigma, void* out, dip_stream_t stream);
/* total_loss.backward() through the network (denoising.ipynb c10:24): dout [C_out][H][W] = dL/d(out).
 * Fills the bound grads[] (overwrite, not accumulate). */
int dip_backward(dip_plan* plan, const void* dout, dip_stream_t stream);
/* dL/d(net_input) of the last dip_backward (plans created with input_grad = 1): dz [C_in][H][W], overwritten.
 * Replaces autograd's gradient of the closure w.r.t. `net_input` when it is optimised (get_params('net,input')). */
int dip_input_grad(dip_plan* plan, void* dz, dip_stream_t stream);

/* torch.nn.MSELoss()(out*mask, target*mask) and its gradient (denoising.ipynb c8:50,c10:23; inpainting.ipynb c17:17).
 * loss: device double (accumulated: zero it first); dout may be NULL; mask [H*W] or NULL. */
int dip_loss_mse(const void* out, const void* target, const void* mask, int channels, int hw, double* loss,
                 void* dout, dip_stream_t stream);
/* net_input = net_input_saved + noise.normal_() * sigma (denoising.ipynb c10:12-13), Philox4x32-10 on device. */
int dip_noise_perturb(const void* z0, void* z, float sigma, uint64_t seed, uint64_t offset, size_t n,
                      dip_stream_t stream);

/* ---- Downsampler.forward and its adjoint (reference: models/downsampler.py:58-71 = nn.ReplicationPad2d(pad) +
 *      nn.Conv2d(C, C, KxK, stride=factor) with the plane-diagonal weight built at models/downsampler.py:44-56;
 *      used as `out_LR = downsampler(out_HR)` in super-resolution.ipynb c10:8).  x: planes [C][H][W]; kern: DEVICE
 *      [K][K] fp32 taps (any of the reference's kernel types; Lanczos-2, K = 16 for factor 4); y: [C][Ho][Wo] with
 *      Ho = dip_lanczos_down_out_size(H, K, factor, pad) = (H + 2 pad - K) / factor + 1.  bwd: dy -> dx (overwrites). */
int dip_lanczos_down_out_size(int n, int K, int factor, int pad);
int dip_lanczos_down_fwd(const void* x, int C, int H, int W, const void* kern, int K, int factor, int pad, void* y,
                         dip_stream_t stream);
int dip_lanczos_down_bwd(const void* dy, int C, int H, int W, const void* kern, int K, int factor, int pad, void* dx,
                         dip_stream_t stream);
/* Runner option for the super-resolution closure (super-resolution.ipynb c10:8-11: total_loss = mse(downsampler(out),
 * img_LR)): dip_run_iterations then computes the loss on the downsampled output; `target` (and `mask`) are
 * [C_out][Ho][Wo].  kern_host: HOST [K][K] fp32 taps, copied; K = 0 / NULL switches the option off. Synchronous setup call. */
int dip_plan_set_downsampler(dip_plan* plan, const float* kern_host, int K, int factor, int pad);

/* ---- torch.optim.Adam(parameters, lr).step() as one multi-tensor launch (utils/common_utils.py:225-230). */
int dip_adam_create(int ntensors, const long long* numel, dip_adam** out);
void dip_adam_destroy(dip_adam* a);
int dip_adam_bind(dip_adam* a, void* const* p, void* const* g, void* const* m, void* const* v);
int dip_adam_step(dip_adam* a, double lr, double beta1, double beta2, double eps, int step, dip_stream_t stream);

/* ---- closure-free runner: `iters` iterations of  noise -> forward -> MSE -> backward -> Adam  entirely on the
 *      device (utils/common_utils.py:227-230 with the lean closure of denoising.ipynb c10).  m, v: Adam state
 *      (ntensors buffers).  Losses (device doubles, one per iteration) are written to loss_hist if non-NULL.
 *      step0 = number of Adam steps already taken.
 *      The runner's Adam step uses torch's defaults: betas (0.9, 0.999), eps 1e-8. */
int dip_run_iterations(dip_plan* plan, dip_adam* adam, const void* z0, const void* target, const void* mask,
                       float sigma, uint64_t seed, int step0, int iters, double lr, void* out, double* loss_hist,
                       dip_stream_t stream);

/* ---- the runner with the rest of the denoising closure (denoising.ipynb c10:8-56) on the device: every iteration, after
 *      the loss and before the Adam step,
 *        1. out_avg = out (first tracked iteration), else out_avg * exp_weight + out * (1 - exp_weight) in torch's fp32
 *           rounding (each scalar rounded to fp32, three separately rounded operations);
 *        2. psnr_target = -10 log10(loss) (c10's psrn_noisy; psrn_masked / psnr_LR for inpainting / super-resolution),
 *           psnr_gt = -10 log10(mean((out - gt)^2)), psnr_gt_sm = the same for the updated out_avg, all in fp64
 *           (skimage compare_psnr, data range 1; unmasked; NaN without gt);
 *        3. back-tracking (c10:41-52) when show_every > 0 and i % show_every != 0: if psnr_target - psnr_last <
 *           -backtrack_db and a snapshot exists, the Adam step starts from the snapshot instead of the parameters (m, v and
 *           the step advance with this iteration's gradient), i stays, fallbacks += 1; otherwise the snapshot becomes the
 *           parameters this iteration's forward used, psnr_last = psnr_target, i += 1.  Elsewhere only i += 1.
 *           BatchNorm running statistics are not restored (the notebook does not restore them either);
 *        4. records[iteration] = {loss, psnr_target, psnr_gt, psnr_gt_sm, i before this iteration, action}, action
 *           0 none, 1 saved, 2 restored.
 *      The state persists across calls; all zero = the notebook's initial globals (i = 0, out_avg = None, last_net = None,
 *      psrn_noisy_last = 0). */
typedef struct {
  const void* gt;        /* [C_out][H][W] clean image, or NULL (psnr_gt / psnr_gt_sm = NaN)                        */
  void* out_avg;         /* [C_out][H][W] fp32: the EMA                                                            */
  void* snapshot;        /* fp32, sum of the Adam tensors' numel, in their order                                   */
  void* state;           /* dip_track_state_bytes() bytes; all zero = the notebook's initial globals               */
  double* records;       /* [iters][6], see above                                                                  */
  double exp_weight;     /* in [0, 1); 0.99 in denoising.ipynb c10 (double: the rounding of 1 - exp_weight is torch's) */
  int show_every;        /* >= 0; 0 = no back-tracking                                                             */
  double backtrack_db;   /* 5 in denoising.ipynb c10:42                                                            */
} dip_track;
size_t dip_track_state_bytes(void);
/* dip_run_iterations with the tracker above; track == NULL is dip_run_iterations.  Invalid fields are refused before
 * anything is launched (dip_last_error() names the field). */
int dip_run_iterations_tracked(dip_plan* plan, dip_adam* adam, const void* z0, const void* target, const void* mask,
                               float sigma, uint64_t seed, int step0, int iters, double lr, void* out, double* loss_hist,
                               const dip_track* track, dip_stream_t stream);

/* ---- test / profiling access to internal NHWC buffers: name e.g. "L0.raw_u"; dims = {rows, cols, ld, channels} */
int dip_plan_buffer(const dip_plan* plan, const char* name, void** ptr, int* dims4);
int dip_plan_num_launches(const dip_plan* plan, int* fwd, int* bwd);
/* CUDA-event brackets around every tensor-core launch (for bench.py's roofline). get_timing drains the records:
 * index 0 = fprop, 1 = dgrad (both tc_conv_kernel), 2 = wgrad (tc_wgrad_kernel); flops are algorithmic (2*M*N*K). */
int dip_plan_set_timing(dip_plan* plan, int enable);
int dip_plan_get_timing(dip_plan* plan, double* ms3, double* flops3, int* launches3);
/* same records one by one (class, algorithmic flops, device ms); returns the number written (<= max_records).
 * Class 3 = k_bn_bwd_apply with a plain gradient source (HBM-bound; `flops` then holds the algorithmic BYTES:
 * read raw + read gradient + write input gradient), class 4 = the other BN-backward apply launches (bytes likewise). */
int dip_plan_get_timing_records(dip_plan* plan, int max_records, int* cls, double* flops, double* ms);

/* ---- single-op entry points (same kernels as the plan; used by the per-kernel parity tests).
 * Convolution of an NHWC fp32 tensor a[a_h][a_w][a_c] with torch OIHW weights w[N][C][k][k]:
 *   d[y][x][n] = bias[n] + sum a[y*stride+offy+r][x*stride+offx+s][c] * w[n][(c+rot)%C][r][s], out-of-range reads = 0.
 * scratch: device buffer of at least dip_op_scratch_bytes(); it holds the packed weights, the weight-gradient partials
 * and, in precision bf16, bf16 copies of the operands.  Operands that do not fit return an error naming the scratch,
 * and nothing is launched. stats (nullable): 2*N fp64
 * accumulators (sum, sum^2), accumulated: element i lives at stats[16*i] (one accumulator per 128-byte line, so the
 * fp64 atomics of neighbouring channels never share an L2 line); the buffer holds 2*N*16 doubles. */
size_t dip_op_scratch_bytes(void);
int dip_op_conv_fprop(const void* a, int a_h, int a_w, int a_c, const void* w, const void* bias, int N, int C, int k,
                      int stride, int offx, int offy, int rot, void* d, int d_h, int d_w, double* stats,
                      int precision, void* scratch, dip_stream_t stream);
/* dgrad on the padded domain: dx[u][v][c] = sum dy[u-r+off][v-s+off][n] w[n][(c+rot)%C][r][s]; off = 0 gives the
 * "full" correlation onto (dy_h + k - 1) x (dy_w + k - 1). */
int dip_op_conv_dgrad(const void* dy, int dy_h, int dy_w, const void* w, int N, int C, int k, int rot, void* dx,
                      int dx_h, int dx_w, int precision, void* scratch, dip_stream_t stream);
/* Input gradient of a 3x3 STRIDE-2 convolution (the adjoint that autograd runs for the down-sampling convs,
 * models/skip.py:64 / models/common.py:120; = ConvTranspose2d(stride 2)), read from dy at its own resolution (tensor
 * cores: its four sub-pixel phases; precision fp32: a stride-1 conv over dy dilated by 2):
 * dx[(2*dy_h+2)][(2*dy_w+2)][C], dx[u][v][c] = sum_{r = u mod 2 .. , s = v mod 2 ..} dy[(u-r)/2][(v-s)/2][n]
 * w[n][(c+rot)%C][r][s]  (every element of dx is written). */
int dip_op_conv_dgrad_s2(const void* dy, int dy_h, int dy_w, const void* w, int N, int C, int rot, void* dx, int precision,
                         void* scratch, dip_stream_t stream);
/* dw[n][(c+rot)%C][r][s] = sum dy[y][x][n] * a[y*stride+offy+r][x*stride+offx+s][c] */
int dip_op_conv_wgrad(const void* dy, int dy_h, int dy_w, const void* a, int a_h, int a_w, int a_c, int N, int C,
                      int k, int stride, int offx, int offy, int rot, void* dw, int precision, void* scratch,
                      dip_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* DIP_H_ */
