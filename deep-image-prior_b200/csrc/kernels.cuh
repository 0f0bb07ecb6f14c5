// Launch wrappers of the HBM-bound kernels of the dip engine (kernels_mem.cu, conv_simt.cu).
// All activations are fp32 NHWC; "ld" is the channel stride of a buffer in floats.  Precision mode bf16 adds bf16 twins (Twin) of
// the tensors the tensor-core kernels read; everything these kernels compute with stays fp32.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

namespace dip {

static constexpr float kBnEps = 1e-5f;
static constexpr long long kNumSms = 132;      // H100 SXM: grid caps of the grid-stride kernels (a few blocks per SM)
static constexpr float kLreluSlope = 0.2f;
// activation of every BN(+act) stage = models.skip's act_fun (models/common.py:76-92); the values are DIP_ACT_* of dip.h
static constexpr int kActLeakyRelu = 0, kActSwish = 1, kActElu = 2, kActNone = 3;
// fp64 accumulators are spread one per 128-byte line (stride in doubles): hundreds of blocks add to them at the end of
// every reduction kernel: neighbouring channels must not share an L2 atomic unit, and each accumulator is split into
// kAccR replicas (same-address atomics serialise) that readers add up
static constexpr int kAccLine = 16;            // one 128-byte line
#ifndef DIP_ACC_R
#define DIP_ACC_R 1
#endif
static constexpr int kAccR = DIP_ACC_R;        // replicas per accumulator (block b adds to replica b % kAccR)
static constexpr int kAccS = kAccLine * kAccR; // stride between consecutive accumulators, in doubles
// value of the accumulator whose replica 0 is *p
__host__ __device__ inline double acc_get(const double* p) {
  double s = p[0];
#pragma unroll
  for (int r = 1; r < kAccR; ++r) s += p[r * kAccLine];
  return s;
}

// Programmatic dependent launch: every kernel of the step calls pdl_trigger() first (the next kernel of the stream may
// be scheduled as SMs drain) and pdl_wait() before it touches global memory (returns once the previous kernel has
// completed and its writes are visible), so the launch latency and the prologue of kernel k+1 overlap the tail of k.
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_enter() { pdl_trigger(); pdl_wait(); }
#endif
inline bool pdl_enabled() {
  static const bool on = getenv("DIP_PDL") != nullptr;  // opt-in: the step is replayed as a CUDA graph anyway
  return on;
}
// kernel<<<grid, block, smem, s>>>(args...) with the programmatic-serialization attribute (and an optional cluster)
template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, int cluster,
                            Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute at[2];
  int n = 0;
  if (pdl_enabled()) {
    at[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  if (cluster > 1) {
    at[n].id = cudaLaunchAttributeClusterDimension;
    at[n].val.clusterDim.x = cluster;
    at[n].val.clusterDim.y = 1;
    at[n].val.clusterDim.z = 1;
    ++n;
  }
  cfg.attrs = at;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// Optional bf16 twin of an NHWC fp32 output (precision mode bf16: the tensor-core kernels read their operands from these).
// Same pixel order as the fp32 tensor; ld = channel stride in bf16 elements (a multiple of 8: TMA needs 16-byte pitches;
// channels between the tensor's depth and ld are never written nor read).  p == nullptr: no twin.
struct Twin {
  uint16_t* p;
  int ld;
};
static constexpr Twin kNoTwin = {nullptr, 0};
// plain NHWC fp32 [npix][ld] (c valid channels, c % 4 == 0) -> bf16 [npix][t.ld]   (single-op entry points)
void launch_cast_bf16(const float* x, int ld, int c, long long npix, Twin t, cudaStream_t s);

// Statistics of one BatchNorm layer: fp64 accumulators, zeroed once per iteration.
//   fwd[0..C)   sum x          fwd[C..2C)   sum x^2
//   bwd[0..C)   sum dz         bwd[C..2C)   sum dz * xhat          (dz = grad wrt BN output)
//   dbias[0..C) sum dx         (grad wrt the conv bias that feeds this BN)
struct BnRef {
  const double* fwd;   // [2*C]
  const float* gamma;  // [C] (torch order)
  const float* beta;   // [C]
  int C;               // channels
  int rot;             // torch channel = (c + rot) % C   (4 for the concat BN: [up|skip] here, [skip|up] in torch)
  float inv_n;         // 1 / (H*W)
};

// RGB head fused into the last BN+activation stage: out[k][p] = sigmoid(b[k] + sum_c w[k][c] * act(bn(raw))[p][c])
struct HeadRef {
  const float* w;      // [K][C] (torch [K][C][1][1])
  const float* b;      // [K]
  int K;               // <= 4
  float* out;          // NCHW [K][H*W]
  int sigmoid;         // 1: nn.Sigmoid behind the head (need_sigmoid=True, skip.py:97-98), 0: the logits are the output
};

// z (NCHW, C x H x W) [+ sigma * noise (NCHW)] -> reflection-padded NHWC [(H+2)][(W+2)][C]
// C = stored depth of dst; c_src (0: C) = depth of z / noise, the remaining channels are written as zeros
// zero_pad = 1: the halo ring is written as zeros (Conv2d(padding=1) instead of ReflectionPad2d(1)); the same switch on
// every launcher below that writes or folds a halo
void launch_input_pad(const float* z, const float* noise, float sigma, float* dst, int C, int H, int W,
                      cudaStream_t s, int c_src = 0, Twin t16 = kNoTwin, int zero_pad = 0);

// generic per-channel sum / sum^2 of a plain NHWC tensor (SIMT-conv path and skinny convs)
void launch_channel_stats(const float* x, int ld, int C, int npix, double* fwd, cudaStream_t s);

// y = f(bn(x)) written plain [H][W][ld_out] or reflection padded [(H+2)][(W+2)][ld_out]; f = the activation act_fun
// (kAct*) when act != 0, else the identity
// dst may be null when a bf16 twin is given (the tensor is then only read by tensor-core kernels)
void launch_bn_act_write(const float* raw, int ld_in, BnRef bn, int H, int W, float* dst, int ld_out, int pad,
                         int act, int act_fun, cudaStream_t s, Twin t16 = kNoTwin, int zero_pad = 0);
// y = f(bn(x)) consumed on the fly by the RGB head (C must be 128); y itself is not materialised
void launch_bn_act_head(const float* raw, BnRef bn, int H, int W, HeadRef head, int act_fun, cudaStream_t s);

// Concat stage:  cat = [ up2x(U)(Cu ch) | f(bn_s(raw_s))(Cs ch) ] at H x W (U is H/2 x W/2, plain, ld = Cu), f = act_fun
struct CatArgs {
  const float* U;      // [H/2][W/2][Cu]
  const float* raw_s;  // [H][W][Cs]
  BnRef bn_s;          // BN of the skip branch
  int Cu, Cs, H, W;
  int bilinear;        // 1 bilinear (align_corners=False), 0 nearest
};
void launch_cat_stats(CatArgs a, double* fwd_cat, int act_fun, cudaStream_t s);
// dst = bn_cat(cat) with reflection pad: [(H+2)][(W+2)][Cu+Cs]
void launch_cat_write(CatArgs a, BnRef bn_cat, float* dst, int act_fun, cudaStream_t s, Twin t16 = kNoTwin, int zero_pad = 0);

// Gradient sources for the BN backward kernels
struct GradSrc {
  int kind;            // 0 plain, 1 fold(padded) (+ skip-conv dgrad), 2 upsample-adjoint, 3 RGB head
  const float* g;      // kind 0: [H][W][ld] (+coff) ; kind 1: padded [(H+2)][(W+2)][ld] ; kind 2: [2H][2W][ld]
  int ld, coff;
  // kind 1: optional second consumer = 1x1 skip conv of the next level: g += sum_n ds[p][n] * w2[n][c]
  const float* ds;     // [H][W][n2] or null
  const float* w2;     // [n2][C]
  int n2;
  // kind 1: optional plain addend (skip=128: the tensor-core dgrad of the next level's skip conv): g += add[p][c]
  const float* add;    // [H][W][ld_add] or null
  int ld_add;
  int bilinear;        // kind 2
  // kind 3: g[p][c] = sum_k dout[k][p] * o[k][p] * (1 - o[k][p]) * wh[k][c]; also accumulates the head's own gradients
  const float* dl4;    // [npix][4] logit gradients dout * o * (1 - o) (launch_head_dlogit)
  const float* wh;     // [K][C]
  int nh;
  // kind 1: adjoint of zero padding (the halo of g is dropped) instead of the reflection fold.  (Placed in the alignment gap
  // after nh: the struct's size and the offsets of the other fields stay those of the reflection-only layout.)
  int zero_pad;
  double* dwh;         // [K][C] fp64 accumulators (reduce pass)
  double* dbh;         // [K]
};

// dl4[p][k] = dout[k][p] * o[k][p] * (1 - o[k][p]) (k < K, else 0); dout / outv are NCHW [K][npix]
//   sigmoid = 0 (need_sigmoid=False): dl4[p][k] = dout[k][p]
void launch_head_dlogit(const float* dout, const float* outv, int K, int npix, float* dl4, cudaStream_t s, int sigmoid = 1);
// dL/dz of the network input (OPT_OVER='input', utils/common_utils.py:47-49), torch layout [C][H][W]:
//   dz[c][i][j] = fold(gp)[i][j][c] + ds[i][j][c]; gp = padded dgrad output of the level-0 stride-2 conv
//   [(H+2)][(W+2)][ld], ds = input gradient of the level-0 skip conv [H][W][ld] (nullable)
void launch_input_grad(const float* gp, const float* ds, int ld, int C, int H, int W, float* dz, cudaStream_t s,
                       int zero_pad = 0);

// BN(+activation) backward. reduce: bwd[0..C) += sum dz, bwd[C..2C) += sum dz*xhat.
// dz = f'(y) * gradient (act != 0; f = act_fun, y = the pre-activation, recomputed from raw) or the gradient itself.
// apply: dx = gamma*rstd*(dz - mean(dz) - xhat*mean(dz*xhat)); writes draw plain [H][W][C]; dbias[c] += sum dx.
void launch_bn_bwd_reduce(const float* raw, int ld_raw, BnRef bn, int act, int act_fun, GradSrc src, int H, int W,
                          double* bwd, cudaStream_t s);
// draw may be null when a bf16 twin is given
void launch_bn_bwd_apply(const float* raw, int ld_raw, BnRef bn, int act, int act_fun, GradSrc src, int H, int W,
                         const double* bwd, float* draw, double* dbias, cudaStream_t s, Twin t16 = kNoTwin);

// In-net 'avg' downsampling (models/common.py:101-105: conv stride 1 + nn.AvgPool2d(2, 2)): y[i][j][c] = mean of the 2 x 2 block
// of x [2h][2w][C]; its adjoint spreads 0.25 * dy to the four positions (optionally also as a bf16 twin; dx may be null then)
void launch_avgpool2(const float* x, int h, int w, int C, float* y, cudaStream_t s);
void launch_avgpool2_bwd(const float* dy, int h, int w, int C, float* dx, cudaStream_t s, Twin t16 = kNoTwin);

// Concat-BN backward (no activation). pcat = the stored BN output (padded [(H+2)][(W+2)][ld], ld = bn_cat.C), from which
// xhat is recovered; gradient = fold of the padded dgrad output gp [(H+2)][(W+2)][ld]; dcat plain [H][W][C].
void launch_cat_bwd_reduce(const float* pcat, BnRef bn_cat, const float* gp, int ld, int H, int W, double* bwd,
                           cudaStream_t s, int zero_pad = 0);
void launch_cat_bwd_apply(const float* pcat, BnRef bn_cat, const float* gp, int ld, int H, int W, const double* bwd,
                          float* dcat, cudaStream_t s, int zero_pad = 0);
// adjoint of the x2 upsampling, once per level: dst[h][w][C] <- D[2h][2w][ld] channels [coff, coff+C)
void launch_upadj(const float* D, int ld, int coff, int h, int w, int C, int bilinear, float* dst, cudaStream_t s);

// Skinny 1x1 convs (N <= 4 outputs): y[p][n] = b[n] + sum_c x[p][c] w[n][c]
//   x: pixel (i,j) at x + (i*x_rs + j)*ldx floats (works for padded interiors)
//   mode 0: y NHWC [H][W][N]; mode 1: y = sigmoid(.) NCHW [N][H][W]; mode 2: NCHW without sigmoid
//   stats (nullable, mode 0): fwd[0..N) += sum y, fwd[N..2N) += sum y^2
//   cw (0: C) = row length of w when the stored depth C is padded (channels >= cw multiply zeros)
void launch_skinny_fwd(const float* x, int ldx, int x_rs, const float* w, const float* b, int C, int N, int H,
                       int W, float* y, int mode, double* stats, cudaStream_t s, int cw = 0);
// backward: dy NHWC [H][W][N] (mode 0) or dout NCHW with sigmoid derivative folded in (mode 1: dy = dout*o*(1-o))
//   dx (optional) plain [H][W][C]; dw[N][C] and db[N] accumulated into fp64 (zeroed by caller)
void launch_skinny_bwd(const float* x, int ldx, int x_rs, const float* w, int C, int N, int H, int W,
                       const float* dy, const float* out_nchw, int mode, float* dx, double* dw, double* db,
                       cudaStream_t s, int cw = 0);

// loss[slot] += mean(m^2 (o - t)^2), dout = 2 m^2 (o - t) / n; mask may be null ([H*W], broadcast over C channels);
// slot = *it_dev if it_dev != null else 0
void launch_mse(const float* out, const float* target, const float* mask, int C, int HW, double* loss, float* dout,
                const int* it_dev, cudaStream_t s);

// z = z0 + sigma * N(0,1)  (Philox4x32-10 + Box-Muller; counter = element index / 4, key = seed,
// stream = offset + *it_dev)
void launch_noise(const float* z0, float* z, float sigma, uint64_t seed, uint64_t offset, const int* it_dev, size_t n,
                  cudaStream_t s);
// runner input in one pass: dst (reflection-padded NHWC [(H+2)][(W+2)][C]) = pad(z0 + sigma * N(0,1)), the same Philox stream
// as launch_noise (W % 4 == 0); channels >= c_src of the stored depth C are written as zeros
void launch_noise_pad(const float* z0, float sigma, uint64_t seed, uint64_t offset, const int* it_dev, float* dst, int C, int H,
                      int W, int c_src, cudaStream_t s, Twin t16 = kNoTwin, int zero_pad = 0);
// it_dev[0] += 1, it_dev[1] += 1 (step / iteration counters of the graph-captured runner)
void launch_advance(int* it_dev, cudaStream_t s);

// Downsampler (super-resolution operator, models/downsampler.py:58-71): planes [C][H][W], taps kern[K][K] (device),
// replication pad `pad`, stride f; output planes [C][Ho][Wo] with Ho = down_out_size(H, K, f, pad).   (downsample.cu)
int down_out_size(int n, int K, int f, int pad);
cudaError_t down_kernels_init();   // per-device function attributes (dynamic shared memory opt-in)
cudaError_t launch_down_fwd(const float* x, int C, int H, int W, const float* kern, int K, int f, int pad, float* y,
                            cudaStream_t s);
// adjoint: dy [C][Ho][Wo] -> dx [C][H][W] (every element written)
cudaError_t launch_down_bwd(const float* dy, int C, int H, int W, const float* kern, int K, int f, int pad, float* dx,
                            cudaStream_t s);

// Adam ---------------------------------------------------------------------------------------------
struct AdamTable {
  float* const* p;
  const float* const* g;
  float* const* m;
  float* const* v;
  const int* blk_tensor;   // per block: tensor index
  const int* blk_start;    // per block: first element
  const int* numel;        // per tensor
  int nblocks;
};
// step (1-based) = step + *it_dev when it_dev != null
void launch_adam(AdamTable t, double lr, double b1, double b2, double eps, int step, const int* it_dev,
                 cudaStream_t s);
int adam_chunk();

// Denoising-closure tracker (denoising.ipynb c10:8-52, dip_track in include/dip.h) ---------------------------------------
// Persistent state; all zero = the notebook's initial globals (i = 0, out_avg = None, last_net = None, psrn_noisy_last = 0).
struct TrackState {
  double psnr_last;   // psrn_noisy_last
  int i;              // the notebook's iteration counter (not advanced by a restore)
  int action;         // this iteration's decision, read by the tracked Adam step: kTrack*
  int has_avg;        // out_avg holds an average (0: the next output is copied)
  int has_snapshot;   // the snapshot holds parameters (last_net is not None)
  int fallbacks;      // restores so far
  int unused;
};
enum { kTrackNone = 0, kTrackSaved = 1, kTrackRestored = 2 };
static constexpr int kTrackRecord = 6;   // doubles per iteration: loss, psnr_target, psnr_gt, psnr_gt_sm, i, action
// out_avg = out (first tracked iteration) or fl(fl(out_avg * w_avg) + fl(out * w_out)); with gt != null the two fp64 sums
// mean((out - gt)^2), mean((out_avg - gt)^2) are accumulated into rec[slot][2], rec[slot][3] with k_mse's reduction
// (slot = *it_dev if it_dev != null else 0; the slot must be zero)
void launch_track_out(const float* out, const float* gt, float* out_avg, const TrackState* st, float w_avg, float w_out,
                      int n, double* rec, const int* it_dev, cudaStream_t s);
// one warp: rec[slot] = {loss[slot], PSNRs of the loss and of the two sums (NaN without gt), i, action}; applies the
// back-tracking rule and updates *st
void launch_track_decide(const double* loss, double* rec, TrackState* st, int show_every, double backtrack_db, int has_gt,
                         const int* it_dev, cudaStream_t s);
// Adam with the tracker's action: st->action == kTrackRestored steps from the snapshot instead of p; kTrackSaved stores the
// p it read into the snapshot.  snapshot: one flat buffer, tensor i at off[i] (the tensors' numel prefix sums).
struct AdamTrack {
  const TrackState* st;
  float* snapshot;
  const long long* off;
};
void launch_adam_track(AdamTable t, double lr, double b1, double b2, double eps, int step, const int* it_dev, AdamTrack tr,
                       cudaStream_t s);

// SIMT fp32 reference convolutions (exact-fp32 mode) ---------------------------------------------------
struct SimtConvArgs {
  const float* A; int a_h, a_w, a_ld, a_c;       // input NHWC (rows, cols, stride, valid channels)
  const float* Wp; int n_rows, c_pad;            // packed weights [tap][n_rows][c_pad]
  float* D; int d_h, d_w, d_ld, d_c;             // output NHWC
  int kh, kw, stride, offx, offy;
  const float* bias;
  int dil = 1;                                   // input dilation (1 or 2): the input the kernel convolves is
                                                 // (dil*a_h) x (dil*a_w), A[i][j] at (dil*i, dil*j) and zeros between
};
void launch_simt_conv(SimtConvArgs a, cudaStream_t s);
struct SimtWgradArgs {
  const float* dY; int h, w;                     // [h][w][dy_ld], n output channels (0 / 0: 128 / 128)
  int dy_ld, n;
  const float* X; int x_h, x_w, x_ld, x_c;
  int kh, kw, stride, offx, offy;
  float* partial; int c_pad;                     // [ksplits][tap][128][c_pad]
  int ksplits;
};
void launch_simt_wgrad(SimtWgradArgs a, cudaStream_t s);

}  // namespace dip
