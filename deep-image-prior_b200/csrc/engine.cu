// dip engine: plan builder (shapes -> HBM buffers, TMA tensor maps, kernel schedule) and the C ABI of
// libdip.so (include/dip.h).  Replaces the execution of the reference's skip network
// (models/skip.py:41-100, module tree interpreted by torch.nn.Sequential) + autograd backward + Adam.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <initializer_list>
#include <map>
#include <string>
#include <vector>

#include "../../include/dip.h"
#include "conv_tc.cuh"
#include "kernels.cuh"

namespace dip {

static thread_local std::string g_err;
static int fail(const std::string& m) {
  g_err = m;
  return -1;
}
#define DIP_CUDA(expr)                                                                                   \
  do {                                                                                                   \
    cudaError_t _e = (expr);                                                                             \
    if (_e != cudaSuccess) return fail(std::string(#expr) + ": " + cudaGetErrorString(_e));              \
  } while (0)
#define DIP_CHECK(expr)        \
  do {                         \
    int _r = (expr);           \
    if (_r != 0) return _r;    \
  } while (0)

// ------------------------------------------------------------------------------------------------ tensor maps
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled g_encode = nullptr;
static int g_num_sms = 0;
static unsigned long long g_inited_mask = 0;   // one bit per device: function attributes (dynamic smem opt-in) are per device

static int engine_init() {
  int dev = 0;
  DIP_CUDA(cudaGetDevice(&dev));
  if (dev >= 64) return fail("dip: device ordinal >= 64 not supported");
  if (g_inited_mask & (1ull << dev)) return 0;
  cudaDeviceProp prop;
  DIP_CUDA(cudaGetDeviceProperties(&prop, dev));
  if (prop.major != 9 || prop.minor != 0)
    return fail("dip requires an sm_90 (H100) device; found sm_" + std::to_string(prop.major * 10 + prop.minor));
  g_num_sms = prop.multiProcessorCount;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  DIP_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
  if (fn == nullptr || q != cudaDriverEntryPointSuccess) return fail("cuTensorMapEncodeTiled not available from the driver");
  g_encode = reinterpret_cast<PFN_encodeTiled>(fn);
  DIP_CUDA(tc_kernels_init());
  DIP_CUDA(down_kernels_init());
  g_inited_mask |= 1ull << dev;
  return 0;
}

static bool is_tc(int prec) { return prec == DIP_PRECISION_TF32 || prec == DIP_PRECISION_BF16; }   // tensor-core paths

static int encode_map(CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_b,
                      const cuuint32_t* box, bool bf16 = false, bool swizzle = true) {
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = g_encode(m, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, rank, const_cast<void*>(base), dims, strides_b, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[256];
    snprintf(buf, sizeof buf, "cuTensorMapEncodeTiled failed (%d): rank %d dims %llu %llu %llu box %u %u %u", (int)r, rank,
             (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)(rank > 2 ? dims[2] : 0), box[0],
             box[1], rank > 2 ? box[2] : 0);
    return fail(buf);
  }
  return 0;
}
// activation [rows][cols][ld] (c valid channels) as the 5-D view (C, px, X, py, Y) used by the conv kernels
// bf16 = true: the tensor holds bf16 (ld in elements); a box row is still 128 bytes = 64 channels
static int map_act5(CUtensorMap* m, const void* base, int rows, int cols, int ld, int c, int stride, int bw, int bh,
                    bool bf16 = false) {
  const cuuint64_t e = bf16 ? 2 : sizeof(float);
  cuuint64_t dims[5], str[4];
  if (stride == 1) {
    dims[0] = c; dims[1] = 1; dims[2] = cols; dims[3] = 1; dims[4] = rows;
    str[0] = ld * e; str[1] = ld * e; str[2] = (cuuint64_t)cols * ld * e; str[3] = (cuuint64_t)cols * ld * e;
  } else {
    dims[0] = c; dims[1] = 2; dims[2] = cols / 2; dims[3] = 2; dims[4] = rows / 2;
    str[0] = ld * e; str[1] = 2 * ld * e; str[2] = (cuuint64_t)cols * ld * e; str[3] = 2 * (cuuint64_t)cols * ld * e;
  }
  cuuint32_t box[5] = {bf16 ? 64u : 32u, 1, (cuuint32_t)bw, 1, (cuuint32_t)bh};
  return encode_map(m, base, 5, dims, str, box, bf16);
}
static int map_act3(CUtensorMap* m, const void* base, int rows, int cols, int ld, int c, int bw, int bh, bool bf16 = false) {
  const cuuint64_t e = bf16 ? 2 : sizeof(float);
  cuuint64_t dims[3] = {(cuuint64_t)c, (cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t str[2] = {ld * e, (cuuint64_t)cols * ld * e};
  cuuint32_t box[3] = {bf16 ? 64u : 32u, (cuuint32_t)bw, (cuuint32_t)bh};
  return encode_map(m, base, 3, dims, str, box, bf16);
}
// activation [rows][cols][ld] (c valid channels, a multiple of the 16-byte group) as the 4-D view (channels of one 16-byte
// group, X, Y, group) read by the patch path of the conv kernel: one box {group, bw + 2, bh + 2, 8 groups} is the input
// patch of one bw x bh tile and 128-byte K block, written unswizzled as [group][patch row][patch col][16 B]
static int map_patch(CUtensorMap* m, const void* base, int rows, int cols, int ld, int c, int bw, int bh, bool bf16) {
  const cuuint64_t e = bf16 ? 2 : sizeof(float);
  const cuuint64_t g = 16 / e;
  cuuint64_t dims[4] = {g, (cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)c / g};
  cuuint64_t str[3] = {ld * e, (cuuint64_t)cols * ld * e, 16};
  cuuint32_t box[4] = {(cuuint32_t)g, (cuuint32_t)bw + 2, (cuuint32_t)bh + 2, 8};
  return encode_map(m, base, 4, dims, str, box, bf16, false);
}
static int map_w2(CUtensorMap* m, const void* base, int rows_total, int kcols, int box_rows, bool bf16 = false) {
  const cuuint64_t e = bf16 ? 2 : sizeof(float);
  cuuint64_t dims[2] = {(cuuint64_t)kcols, (cuuint64_t)rows_total};
  cuuint64_t str[1] = {kcols * e};
  cuuint32_t box[2] = {bf16 ? 64u : 32u, (cuuint32_t)box_rows};
  return encode_map(m, base, 2, dims, str, box, bf16);
}

static void pick_tile(int w, int h, int* bw, int* bh) {
  const int cand[5][2] = {{128, 1}, {64, 2}, {32, 4}, {16, 8}, {8, 16}};
  long long best = -1;
  for (int i = 0; i < 5; ++i) {
    const long long cw = (w + cand[i][0] - 1) / cand[i][0] * cand[i][0];
    const long long ch = (h + cand[i][1] - 1) / cand[i][1] * cand[i][1];
    // prefer square-ish tiles on ties (smaller halo re-reads for 3x3 taps)
    const long long cost = cw * ch * 64 + (cand[i][0] + cand[i][1]);
    if (best < 0 || cost < best) { best = cost; *bw = cand[i][0]; *bh = cand[i][1]; }
  }
}
static int round_up(int x, int m) { return (x + m - 1) / m * m; }
// ------------------------------------------------------------------------------------------------ enqueue recorder
// Optional CUDA-event brackets around the timed launches (bench.py roofline: algorithmic FLOPs / device time).
struct Timer {
  bool on = false;
  std::vector<cudaEvent_t> pool;
  size_t used = 0;
  struct Rec { int cls; double flops; size_t e0, e1; };
  std::vector<Rec> recs;
  size_t get(cudaStream_t s) {
    if (used == pool.size()) { cudaEvent_t e; cudaEventCreate(&e); pool.push_back(e); }
    cudaEventRecord(pool[used], s);
    return used++;
  }
  void reset() { used = 0; recs.clear(); }
};
// Every operation a pass enqueues (kernel launch, memset, copy) goes through one Recorder: it counts them, and brackets
// those with a timing class when timing is on.
struct Recorder {
  Timer* timer = nullptr;
  int n = 0;   // operations enqueued since the pass reset it
};
// Timing classes: 0 fprop, 1 dgrad, 2 wgrad (the record carries the algorithmic FLOPs); HBM-bound launches are class
// 16 + 8 * kernel id + sub-kind, and the record then carries the launch's ALGORITHMIC bytes (unique elements its contract
// reads + writes, x 4 B; SURVEY.md 8d) -- bench.py's HBM rooflines.  kUntimed: counted only.
enum HbmId { H_INPUT_PAD = 0, H_NOISE, H_SKINNY_FWD, H_BN_ACT_WRITE, H_BN_ACT_HEAD, H_CAT_STATS, H_CAT_WRITE, H_BN_BWD_REDUCE,
             H_BN_BWD_APPLY, H_CAT_BWD_REDUCE, H_CAT_BWD_APPLY, H_UPADJ, H_SKINNY_BWD, H_MSE, H_ADAM, H_HEAD_DLOGIT, H_DOWN_FWD,
             H_DOWN_BWD, H_PACK, H_WGRAD_REDUCE, H_TRACK_OUT, H_TRACK_DECIDE, H_ADAM_TRACK };
static constexpr int kUntimed = -1;
static int hbm(HbmId id, int sub) { return 16 + 8 * (int)id + sub; }
struct EnqScope {
  Timer* t; int cls; double flops; size_t e0 = 0; cudaStream_t s;
  EnqScope(Recorder* r, int cls_, double flops_, cudaStream_t s_)
      : t(r != nullptr && cls_ != kUntimed && r->timer->on ? r->timer : nullptr), cls(cls_), flops(flops_), s(s_) {
    if (r != nullptr) r->n++;
    if (t) e0 = t->get(s);
  }
  ~EnqScope() { if (t) { size_t e1 = t->get(s); t->recs.push_back({cls, flops, e0, e1}); } }
};
// enqueues `stmt` (one operation) through the recorder `rec` (nullptr: neither counted nor timed)
#define ENQ(rec, cls, flops, s, stmt)                                 \
  do {                                                                \
    EnqScope _es((rec), (cls), (double)(flops), (s));                 \
    stmt;                                                             \
  } while (0)

// ------------------------------------------------------------------------------------------------ weight pack and split-K sum
// Every convolution, in the plan and in the single-op entry points, packs its weights through k_pack_table and sums its
// split-K weight-gradient partials through k_wgrad_unpack_table.
struct PackEntry {
  const float* w; float* dst_f; float* dst_d;
  int N, C, k, rot, n_rows, c_pad, c_rows;
  int Ctot, coff;   // weight has Ctot input channels; this entry packs engine channels [coff, coff + C)
  int s2;           // tensor-core dgrad pack of a stride-2 3x3 conv: taps in sub-pixel phase order (kS2Taps), not flipped
  int bf16;         // packs hold bf16 (same buffers); the fprop pack then has rows of c_pad16 (multiple of 64) channels
  int c_pad16;
  int n_pad;        // columns of the dgrad pack: N rounded up to 32 (bf16: to 64)
};
// packed tap t of the 4-phase stride-2 dgrad -> filter tap r * 3 + s.  Phase (a, b) = parity of the padded gradient pixel;
// its taps are r in {2, 0} (a = 0: dY rows i-1, i) or {1} (a = 1), same for s.  Phases in the order (0,0) (0,1) (1,0) (1,1).
__constant__ int kS2Taps[9] = {2 * 3 + 2, 2 * 3 + 0, 0 * 3 + 2, 0 * 3 + 0,   // (0,0): (r', s') = (0,0) (0,1) (1,0) (1,1)
                               2 * 3 + 1, 0 * 3 + 1,                           // (0,1): s = 1
                               1 * 3 + 2, 1 * 3 + 0,                           // (1,0): r = 1
                               1 * 3 + 1};                                     // (1,1)
__global__ void k_pack_table(const PackEntry* __restrict__ tab) {
  pdl_enter();
  const PackEntry e = tab[blockIdx.y];
  const int taps = e.k * e.k;
  const int c_pad = e.bf16 ? e.c_pad16 : e.c_pad;
  __nv_bfloat16* const f16 = reinterpret_cast<__nv_bfloat16*>(e.dst_f);
  __nv_bfloat16* const d16 = reinterpret_cast<__nv_bfloat16*>(e.dst_d);
  const long long nf = e.dst_f != nullptr ? (long long)taps * e.n_rows * c_pad : 0;
  const long long nd = e.dst_d != nullptr ? (long long)taps * e.c_rows * e.n_pad : 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nf + nd; i += (long long)gridDim.x * blockDim.x) {
    if (i < nf) {
      const int c = (int)(i % c_pad), n = (int)((i / c_pad) % e.n_rows), tap = (int)(i / ((long long)c_pad * e.n_rows));
      float v = 0.f;
      if (n < e.N && c < e.C) v = e.w[((long long)n * e.Ctot + (c + e.coff + e.rot) % e.Ctot) * taps + tap];
      if (e.bf16) f16[i] = __float2bfloat16_rn(v); else e.dst_f[i] = v;
    } else {
      const long long j = i - nf;
      const int n = (int)(j % e.n_pad), c = (int)((j / e.n_pad) % e.c_rows), tapf = (int)(j / ((long long)e.n_pad * e.c_rows));
      const int tap = e.s2 ? kS2Taps[tapf] : taps - 1 - tapf;
      float v = 0.f;
      if (n < e.N && c < e.C) v = e.w[((long long)n * e.Ctot + (c + e.coff + e.rot) % e.Ctot) * taps + tap];
      if (e.bf16) d16[j] = __float2bfloat16_rn(v); else e.dst_d[j] = v;
    }
  }
}
// split-K partials [ks][tap][128][cols] of a weight gradient -> OIHW gradient, one entry per conv (the tensor-core plan
// sums all of them in one launch per backward pass, the fp32-mode plan and the single-op wgrad one entry after each
// wgrad); the split-K slices are summed in index order, so the gradient is the same on every run
struct UnpackEntry {
  const float* acc; float* dw;
  int N, C, taps, rot, cols, Ctot, coff, ks;   // cols: row stride of the partials (ConvOp::part_cols)
};
__global__ void k_wgrad_unpack_table(const UnpackEntry* __restrict__ tab) {
  pdl_enter();
  const UnpackEntry e = tab[blockIdx.y];
  const int total = e.N * e.C * e.taps;   // dw elements this entry owns: (n, engine channel c, tap)
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int tap = i % e.taps, c = (i / e.taps) % e.C, n = i / (e.taps * e.C);
    const size_t split = (size_t)e.taps * 128 * e.cols;
    const float* src = e.acc + ((size_t)tap * 128 + n) * e.cols + c;
    float v = 0.f;
    for (int k = 0; k < e.ks; ++k) v += src[k * split];
    e.dw[((size_t)n * e.Ctot + (c + e.coff + e.rot) % e.Ctot) * e.taps + tap] = v;
  }
}
// ------------------------------------------------------------------------------------------------ conv op
// CTAs per pixel tile (output channels split across them) for launches with fewer tiles than SMs: n_rows % (32 * split) == 0
static int pick_nsplit(int tiles, int n_rows) {
  int sp = 1;
  while (sp * 2 <= 4 && tiles * sp * 2 <= g_num_sms && n_rows % (32 * sp * 2) == 0) sp *= 2;
  return sp;
}
static void fit_stages(TcConvParams& p) {
  p.stages = p.patch ? 8 : 6;
  while (tc_conv_smem_bytes(p) > 232448 && p.stages > 2) p.stages--;
}
struct ConvOp {
  Recorder* rec = nullptr;   // the plan's; the single-op entry points count and time nothing
  double alg_flops() const { return 2.0 * out_h * out_w * (double)N * C * k * k; }
  // N output channels (a multiple of 8, <= 128: num_channels_down / num_channels_up of the level), C input channels
  int N = 128, C = 0, k = 1, stride = 1, rot = 0;
  int Np = 128;      // fprop GEMM N: N rounded up to 16 (rows per tap of the fprop pack; rows >= N are zero)
  int n_pad = 128;   // dgrad K extent per tap: N rounded up to 32 (columns of the dgrad pack), n_pad16: to 64 (bf16)
  int n_pad16 = 128;
  // An op may cover a SLICE [coff, coff + C) of the (engine-order) input channels of a wider convolution whose weight has
  // Ctot input channels (the 256-channel up conv of the skip=128 configuration: fprop runs as one op with 8 K blocks,
  // dgrad / wgrad as two 128-channel halves -- the register accumulators hold at most 160 columns).  Ctot == 0: the op is
  // the whole conv.
  int Ctot = 0, coff = 0;
  bool do_fprop = true, do_wgrad = true;
  int dg_ld = 0;   // channel stride of dg_out (0: C)
  int c_pad = 0;   // fprop K extent per tap (multiple of 32)
  int crows = 0;   // dgrad GEMM N (input channels rounded to 16)
  // precision mode bf16: the tensor-core kernels read bf16 twins of the conv input / of dY (written by the producer kernels
  // next to -- or instead of -- the fp32 tensors) and bf16 weight packs; outputs and accumulators stay fp32
  bool bf16 = false;
  int c_pad16 = 0;                                   // fprop K extent per tap in bf16 (multiple of 64)
  const uint16_t* in16 = nullptr; int in_ld16 = 0;   // twin of `in`
  const uint16_t* dy16 = nullptr;                    // twin of `dy`
  // forward: in -> out [out_h][out_w][N]
  const float* in = nullptr; int in_rows = 0, in_cols = 0, in_ld = 0; int offx = 0, offy = 0;
  float* out = nullptr; int out_h = 0, out_w = 0;
  double* stats = nullptr;
  float* wp_f = nullptr; float* wp_d = nullptr;
  // dY [out_h][out_w][N]: the gradient of `out`, read by the dgrad and the wgrad
  const float* dy = nullptr;
  // dgrad: dY -> dg_out [dg_out_h][dg_out_w][C]
  bool has_dgrad = false;
  // input gradient of a stride-2 3x3 conv, read from dY at its own resolution: the tensor-core kernel runs its 4 sub-pixel
  // phases, the SIMT kernel (fp32 mode) a stride-1 conv over dY dilated by 2
  bool dg_s2 = false;
  float* dg_out = nullptr; int dg_out_h = 0, dg_out_w = 0; int dg_off = 0;
  // wgrad: split-K partials [part_ks][tap][128][part_cols] (the tensor-core plan gives every conv its own; the fp32-mode
  // plan shares one area between all convs), summed into the gradient by one UnpackEntry per conv
  float* partial = nullptr;
  const UnpackEntry* unpack = nullptr;   // launched right after the wgrad; nullptr: the plan sums every entry at the end
  // param slots
  int p_w = -1, p_b = -1;
  TcConvParams fp{}, dg{};   // what the launches run: the general form, or its stride-1 3x3 patch form
  TcWgradParams wg{};

  void set_shapes() {
    c_pad = round_up(C, 32);
    c_pad16 = round_up(C, 64);
    crows = round_up(C, 16);
    Np = round_up(N, 16); n_pad = round_up(N, 32); n_pad16 = round_up(N, 64);
    if (Ctot == 0) Ctot = C;
    if (dg_ld == 0) dg_ld = C;
  }
  size_t wp_f_elems() const { return (size_t)k * k * Np * c_pad; }
  size_t wp_d_elems() const { return (size_t)k * k * crows * n_pad; }
  // accumulator columns of the tensor-core weight gradient (wgmma N, row stride of its partials): c_pad, except 136 for
  // 128 < C <= 136 (the 128 + 4 channel concat convs), which would otherwise multiply 24 zero columns of every 160
  int wg_cols() const { return C > 128 && C <= 136 ? 136 : c_pad; }
  // work items per filter tap: about one item per SM of an H100 SXM over all taps (every item writes a [128][wg_cols] partial
  // slice, so more items than SMs only add traffic).  A constant, not the device's count: the plan's size is known
  // without a device, and the split -- hence the summation order of the gradient -- is the same on every device.
  int tc_ksplits() const {
    const int blocks = out_h * ((out_w + kWgradKp - 1) / kWgradKp);
    int ks = static_cast<int>(kNumSms) / (k * k);
    if (ks > blocks) ks = blocks;
    return ks < 1 ? 1 : ks;
  }
  int simt_ksplits() const { return out_h < 64 ? out_h : 64; }   // row ranges of the SIMT weight gradient
  int part_ks(int prec) const { return is_tc(prec) ? tc_ksplits() : simt_ksplits(); }
  int part_cols(int prec) const { return is_tc(prec) ? wg_cols() : c_pad; }
  size_t partial_elems(int prec) const { return (size_t)part_ks(prec) * k * k * 128 * part_cols(prec); }
  PackEntry pack_entry(int prec, const float* w) const {
    PackEntry e{};
    e.w = w; e.dst_f = do_fprop ? wp_f : nullptr; e.dst_d = has_dgrad ? wp_d : nullptr;
    e.N = N; e.C = C; e.k = k; e.rot = rot; e.n_rows = Np; e.c_pad = c_pad; e.c_rows = crows;
    e.Ctot = Ctot; e.coff = coff; e.s2 = dg_s2 && is_tc(prec) ? 1 : 0;   // (the SIMT dgrad reads flipped taps)
    e.bf16 = bf16 ? 1 : 0; e.c_pad16 = c_pad16; e.n_pad = bf16 ? n_pad16 : n_pad;
    return e;
  }
  UnpackEntry unpack_entry(int prec, float* dw) const {
    return UnpackEntry{partial, dw, N, C, k * k, rot, part_cols(prec), Ctot, coff, part_ks(prec)};
  }

  // Replaces the general form g of a stride-1 3x3 conv by its patch form (tc_conv_patch_kernel): the same tiles, weights,
  // output and N split, the activation [rows][cols][ld] (kc K channels) through the 4-D patch map.  It applies when the tile
  // is 8 or 16 pixels wide, the K channels fill whole 16-byte groups (TMA zero-fills the patch past the channel extent only
  // in whole groups) and one patch per K block fits in shared memory beside at least two weight stages; otherwise g stays
  // as it is.  Both forms compute the same sums in the same order.
  int patch_form(TcConvParams& g, const void* act, int rows, int cols, int ld, int kc) {
    if ((g.bw != 8 && g.bw != 16) || kc % (bf16 ? 8 : 4) != 0 || g.kblocks > kPatchMaxKb) return 0;
    TcConvParams t = g;
    t.patch = 1;
    fit_stages(t);
    if (tc_conv_smem_bytes(t) > 232448) return 0;
    DIP_CHECK(map_patch(&t.tmA, act, rows, cols, ld, kc, g.bw, g.bh, bf16));
    g = t;
    return 0;
  }
  int build_tc() {
    // ---- fprop
    int bw, bh;
    fp = TcConvParams{};
    if (do_fprop) {
      pick_tile(out_w, out_h, &bw, &bh);
      DIP_CHECK(bf16 ? map_act5(&fp.tmA, in16, in_rows, in_cols, in_ld16, C, stride, bw, bh, true)
                     : map_act5(&fp.tmA, in, in_rows, in_cols, in_ld, C, stride, bw, bh));
      fp.n_split = pick_nsplit(((out_w + bw - 1) / bw) * ((out_h + bh - 1) / bh), Np);
      DIP_CHECK(map_w2(&fp.tmB, wp_f, k * k * Np, bf16 ? c_pad16 : c_pad, Np / fp.n_split, bf16));
      DIP_CHECK(map_act3(&fp.tmD, out, out_h, out_w, N, N, bw, bh));
      fp.tiles_x = (out_w + bw - 1) / bw; fp.tiles_y = (out_h + bh - 1) / bh;
      fp.bw = bw; fp.bh = bh; fp.out_w = out_w; fp.out_h = out_h;
      fp.kh = fp.kw = k; fp.stride = stride; fp.offx = offx; fp.offy = offy;
      fp.bf16 = bf16 ? 1 : 0;
      fp.kblocks = bf16 ? c_pad16 / 64 : c_pad / 32;
      fp.n_mma = Np / fp.n_split; fp.n_chunks = (fp.n_mma + 31) / 32;
      fp.n_valid = N;
      fp.bias = nullptr; fp.stats = stats; fp.stats_ld = N;
      fit_stages(fp);
      if (k == 3 && stride == 1)
        DIP_CHECK(bf16 ? patch_form(fp, in16, in_rows, in_cols, in_ld16, C) : patch_form(fp, in, in_rows, in_cols, in_ld, C));
    }
    // ---- dgrad: K = the N channels of dY.  Stride 2: the 4 sub-pixel phases over the (dg_out_h / 2) x (dg_out_w / 2)
    // positions of each parity class of the padded gradient
    dg = TcConvParams{};
    if (has_dgrad) {
      const int gh = dg_s2 ? dg_out_h / 2 : dg_out_h, gw = dg_s2 ? dg_out_w / 2 : dg_out_w;
      pick_tile(gw, gh, &bw, &bh);
      DIP_CHECK(bf16 ? map_act5(&dg.tmA, dy16, out_h, out_w, N, N, 1, bw, bh, true)
                     : map_act5(&dg.tmA, dy, out_h, out_w, N, N, 1, bw, bh));
      dg.tiles_x = (gw + bw - 1) / bw; dg.tiles_y = (gh + bh - 1) / bh;
      dg.n_split = pick_nsplit((dg_s2 ? 4 : 1) * dg.tiles_x * dg.tiles_y, crows);
      DIP_CHECK(map_w2(&dg.tmB, wp_d, k * k * crows, bf16 ? n_pad16 : n_pad, crows / dg.n_split, bf16));
      DIP_CHECK(dg_s2 ? map_act5(&dg.tmD, dg_out, dg_out_h, dg_out_w, dg_ld, C, 2, bw, bh)   // parity view of the padded gradient
                      : map_act3(&dg.tmD, dg_out, dg_out_h, dg_out_w, dg_ld, C, bw, bh));
      dg.bw = bw; dg.bh = bh; dg.out_w = gw; dg.out_h = gh;
      dg.stride = 1;
      if (dg_s2) {
        dg.kh = dg.kw = 2; dg.offx = dg.offy = -1;
        dg.nphase = 4;
        int t0 = 0;
        for (int a = 0; a < 2; ++a)
          for (int b = 0; b < 2; ++b) {
            TcConvParams::Phase& q = dg.phs[a * 2 + b];
            q.kh = 2 - a; q.kw = 2 - b; q.offy = a == 0 ? -1 : 0; q.offx = b == 0 ? -1 : 0; q.tap0 = t0; q.opx = b; q.opy = a;
            t0 += q.kh * q.kw;
          }
      } else {
        dg.kh = dg.kw = k; dg.offx = dg.offy = dg_off;
      }
      dg.bf16 = bf16 ? 1 : 0;
      dg.kblocks = bf16 ? n_pad16 / 64 : n_pad / 32;
      dg.n_mma = crows / dg.n_split; dg.n_chunks = (dg.n_mma + 31) / 32;
      fit_stages(dg);
      if (!dg_s2 && k == 3)
        DIP_CHECK(bf16 ? patch_form(dg, dy16, out_h, out_w, N, N) : patch_form(dg, dy, out_h, out_w, N, N));
    }
    // ---- wgrad
    wg = TcWgradParams{};
    if (!do_wgrad) return 0;
    wg.bf16 = bf16 ? 1 : 0;
    DIP_CHECK(bf16 ? map_act3(&wg.tmY, dy16, out_h, out_w, N, N, kWgradKp, 1, true)
                   : map_act3(&wg.tmY, dy, out_h, out_w, N, N, kWgradKp, 1));
    DIP_CHECK(bf16 ? map_act5(&wg.tmX, in16, in_rows, in_cols, in_ld16, C, stride, kWgradKp, 1, true)
                   : map_act5(&wg.tmX, in, in_rows, in_cols, in_ld, C, stride, kWgradKp, 1));
    wg.partial = partial;
    wg.kh = wg.kw = k; wg.stride = stride; wg.offx = offx; wg.offy = offy;
    wg.px_blocks_x = (out_w + kWgradKp - 1) / kWgradKp;
    wg.px_blocks = out_h * wg.px_blocks_x;
    wg.c_chunks = bf16 ? c_pad16 / 64 : c_pad / 32;
    wg.n_cols = wg_cols();
    wg.ksplits = tc_ksplits();
    wg.stages = 6;
    while (tc_wgrad_smem_bytes(wg) > 232448 && wg.stages > 1) wg.stages--;
    if (tc_wgrad_smem_bytes(wg) > 232448) return fail("wgrad stage does not fit in shared memory");
    return 0;
  }

  int run_fprop(int prec, const float* bias, cudaStream_t s) {
    if (is_tc(prec)) {
      TcConvParams p = fp;
      p.bias = bias;
      ENQ(rec, 0, alg_flops(), s, DIP_CUDA(tc_conv_launch(p, g_num_sms, s)));
    } else {
      SimtConvArgs a{};
      a.A = in; a.a_h = in_rows; a.a_w = in_cols; a.a_ld = in_ld; a.a_c = C;
      a.Wp = wp_f; a.n_rows = Np; a.c_pad = c_pad;
      a.D = out; a.d_h = out_h; a.d_w = out_w; a.d_ld = N; a.d_c = N;
      a.kh = a.kw = k; a.stride = stride; a.offx = offx; a.offy = offy; a.bias = bias;
      ENQ(rec, kUntimed, 0, s, launch_simt_conv(a, s));
      if (stats != nullptr) ENQ(rec, kUntimed, 0, s, launch_channel_stats(out, N, N, out_h * out_w, stats, s));
      DIP_CUDA(cudaGetLastError());
    }
    return 0;
  }
  int run_dgrad(int prec, cudaStream_t s) {
    if (is_tc(prec)) {
      ENQ(rec, 1, alg_flops(), s, DIP_CUDA(tc_conv_launch(dg, g_num_sms, s)));
    } else {
      SimtConvArgs a{};
      a.A = dy; a.a_h = out_h; a.a_w = out_w; a.a_ld = N; a.a_c = N; a.dil = dg_s2 ? 2 : 1;
      a.Wp = wp_d; a.n_rows = crows; a.c_pad = n_pad;
      a.D = dg_out; a.d_h = dg_out_h; a.d_w = dg_out_w; a.d_ld = dg_ld; a.d_c = C;
      a.kh = a.kw = k; a.stride = 1; a.offx = a.offy = dg_off; a.bias = nullptr;
      ENQ(rec, kUntimed, 0, s, launch_simt_conv(a, s));
      DIP_CUDA(cudaGetLastError());
    }
    return 0;
  }
  // Every split-K work item of the weight gradient writes its own slice of `partial`; `unpack` (when set) then sums the
  // slices into the OIHW gradient.
  int run_wgrad(int prec, cudaStream_t s) {
    static const bool dbg_skip = getenv("DIP_DBG_SKIP_WGRAD") != nullptr;   // timing diagnostic only: gradients are wrong
    if (dbg_skip) return 0;
    if (is_tc(prec)) {
      ENQ(rec, 2, alg_flops(), s, DIP_CUDA(tc_wgrad_launch(wg, s)));
    } else {
      SimtWgradArgs a{};
      a.dY = dy; a.h = out_h; a.w = out_w; a.dy_ld = N; a.n = N;
      a.X = in; a.x_h = in_rows; a.x_w = in_cols; a.x_ld = in_ld; a.x_c = C;
      a.kh = a.kw = k; a.stride = stride; a.offx = offx; a.offy = offy;
      a.partial = partial; a.c_pad = c_pad; a.ksplits = simt_ksplits();
      ENQ(rec, kUntimed, 0, s, launch_simt_wgrad(a, s));
    }
    if (unpack != nullptr)
      ENQ(rec, hbm(H_WGRAD_REDUCE, 0), ((double)part_ks(prec) + 1.0) * k * k * 128.0 * part_cols(prec) * sizeof(float), s,
          launch_k(k_wgrad_unpack_table, dim3(64, 1), dim3(256), 0, s, 1, unpack));
    DIP_CUDA(cudaGetLastError());
    return 0;
  }
};

// ------------------------------------------------------------------------------------------------ table kernels
struct CvtEntry {
  const double* src; float* dst; int n, rot;
  int row, row_ld;   // dst rows of `row` elements come from accumulator rows of `row_ld` (0: contiguous)
};
__global__ void k_cvt_table(const CvtEntry* __restrict__ tab) {
  pdl_enter();
  const CvtEntry e = tab[blockIdx.x];
  for (int i = threadIdx.x; i < e.n; i += blockDim.x) {
    const int si = e.row > 0 ? (i / e.row) * e.row_ld + i % e.row : i;
    e.dst[(i + e.rot) % e.n] = (float)acc_get(e.src + (size_t)si * kAccS);
  }
}
struct RunEntry {
  const double* fwd; float* rm; float* rv; void* nb; int C, rot; float n; int nb_is_float;
};
__global__ void k_running_table(const RunEntry* __restrict__ tab) {
  pdl_enter();
  const RunEntry e = tab[blockIdx.x];
  if (e.rm == nullptr) return;
  for (int c = threadIdx.x; c < e.C; c += blockDim.x) {
    const int ct = (c + e.rot) % e.C;
    const double m = acc_get(e.fwd + c * kAccS) / e.n;
    double var = acc_get(e.fwd + (e.C + c) * kAccS) / e.n - m * m;
    if (var < 0) var = 0;
    const double unb = e.n > 1.f ? var * e.n / (e.n - 1.0) : var;
    e.rm[ct] = 0.9f * e.rm[ct] + 0.1f * (float)m;
    e.rv[ct] = 0.9f * e.rv[ct] + 0.1f * (float)unb;
  }
  if (threadIdx.x == 0 && e.nb != nullptr) {
    // Module.type(torch.cuda.FloatTensor) (every notebook does this) also casts num_batches_tracked to float32
    if (e.nb_is_float) *reinterpret_cast<float*>(e.nb) += 1.f; else *reinterpret_cast<long long*>(e.nb) += 1;
  }
}

// ------------------------------------------------------------------------------------------------ plan
struct Arena {
  uint8_t* base;
  size_t off = 0;
  template <typename T>
  T* get(size_t n) {
    off = (off + 255) & ~size_t(255);
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += n * sizeof(T);
    return p;
  }
};
struct BufInfo {
  void* ptr; int rows, cols, ld, c;
};
struct BnLayer {
  int C = 0, rot = 0; float n = 1.f;
  double* fwd = nullptr; double* bwd = nullptr; double* dbias = nullptr;
  int p_gamma = -1, p_beta = -1, p_bias = -1, idx = -1;
};
struct Level {
  int H, W, h, w, Cin;   // Cin: stored depth of the level input (power of two >= 4)
  int Cin_act;           // depth of the conv weights that read it (differs at level 0 for input depths like 3)
  int bilinear;          // x2 upsampling into this level: 1 bilinear, 0 nearest (skip.py:81, upsample_mode[i])
  // channel widths (models/skip.py:5-7): nd = num_channels_down[l] (both down convs), nu = num_channels_up[l] (up conv and 1x1),
  // ns = num_channels_skip[l], cu = depth of the tensor upsampled into this level's concat (nu of the level below, or nd at
  // the deepest level).  128 / 128 / {0, 4, 128} / 128 in every BASELINE configuration.
  int nd = 128, nu = 128, ns = 0, cu = 128;
  // downsample_mode 'avg': the first down conv runs at stride 1 into rawF [H][W][nd], raw_d1 = AvgPool2d(2, 2)(rawF);
  // dRawF [H][W][nd] = the pooling adjoint of dRaw_d1 (input of that conv's dgrad / wgrad)
  float *rawF = nullptr, *dRawF = nullptr;
  uint16_t* dRawF16 = nullptr;
  float *Pin, *raw_s, *raw_d1, *P_d1, *raw_d2, *P_d2, *P_cat, *raw_u, *A_u, *raw_v, *U;
  // bf16 twins (precision mode bf16; ld = the fp32 tensor's depth rounded up to 8)
  uint16_t *Pin16 = nullptr, *P_d1_16 = nullptr, *P_d2_16 = nullptr, *P_cat16 = nullptr, *A_u16 = nullptr;
  uint16_t *dRaw_v16 = nullptr, *dRaw_u16 = nullptr, *dRaw_d2_16 = nullptr, *dRaw_d1_16 = nullptr, *dRaw_s16 = nullptr;
  int Pin_ld16 = 0, cat_ld16 = 0;
  float *dUp;  // [h][w][128] adjoint of the upsampling applied to dCat
  float *dS;   // skip=128: [H][W][Cin] input gradient of the (tensor-core) skip conv, levels > 0
  float *dRaw_v, *dA_u, *dRaw_u, *dP_cat, *dCat, *dRaw_s, *dRaw_d2, *dP_d1, *dRaw_d1, *dPin;
  BnLayer bn_s, bn_d1, bn_d2, bn_cat, bn_u, bn_v;
  int p_skip_w, p_skip_b;
  double* dw_s;
  ConvOp d1, d2, up, c11;
  ConvOp sk, up_a, up_b;   // skip=128 only: 1x1 skip conv Cin -> 128; channel halves of the 256 -> 128 up conv (dgrad / wgrad)
};

}  // namespace dip

using namespace dip;

struct dip_plan {
  dip_net_desc desc;
  int H, W;
  int zero_pad = 0;   // dip_plan_opts.pad_mode == DIP_PAD_ZERO: conv-input halos hold zeros (Conv2d(padding=1))
  int act_fun = DIP_ACT_LEAKY_RELU;   // dip_plan_opts.act_fun: the activation of every BN(+act) stage (kAct*)
  bool dry = false;
  uint8_t* ws = nullptr;
  size_t ws_bytes = 0;
  std::vector<Level> lv;
  std::vector<long long> numel;
  std::vector<float*> params, grads;
  std::vector<void*> running;
  std::vector<BnLayer*> bns;
  std::vector<ConvOp*> convs;
  std::map<std::string, BufInfo> bufs;
  // head
  int p_head_w = -1, p_head_b = -1;
  double* dw_head = nullptr; double* db_head = nullptr; double* db_scratch = nullptr;
  float* out_saved = nullptr;  // [C_out][H][W] (sigmoid output, needed by backward)
  // accumulators
  double* acc_fwd = nullptr; size_t acc_fwd_n = 0;
  double* acc_bwd = nullptr; size_t acc_bwd_n = 0;
  float* partial = nullptr;
  // runner scratch
  float* zbuf = nullptr; float* dout = nullptr; float* dl4 = nullptr;
  // super-resolution operator applied between the network output and the loss (dip_plan_set_downsampler)
  static constexpr int kDownMaxK = 64;
  float* ds_kern = nullptr;      // [K][K] taps
  float* ds_y = nullptr;         // [C_out][Ho][Wo] downsampled output
  float* ds_dy = nullptr;        // [C_out][Ho][Wo] dL/d(ds_y)
  int ds_K = 0, ds_f = 1, ds_pad = 0, ds_Ho = 0, ds_Wo = 0;
  static constexpr int kLossRing = 65536;
  double* loss_ring = nullptr;   // [kLossRing] loss slots of the runner when the caller passes no history buffer
  int* it_dev = nullptr;         // [2] device counters: {global Adam step, iteration index of this call}
  // identity of everything the captured step bakes in; compared field by field (the struct has padding).  adam_id is a
  // process-wide serial number: a new dip_adam allocated at the address of a destroyed one must not match.
  struct GraphKey {
    const void *z0 = nullptr, *target = nullptr, *mask = nullptr, *out = nullptr, *slots = nullptr;
    unsigned long long adam_id = 0, adam_bind = 0;
    float sigma = 0.f; uint64_t seed = 0; double lr = 0.0;
    dip_track track{};   // all zero when the runner is untracked (a tracker always has out_avg != NULL)
    bool operator==(const GraphKey& o) const {
      const dip_track &a = track, &b = o.track;
      return z0 == o.z0 && target == o.target && mask == o.mask && out == o.out && slots == o.slots && adam_id == o.adam_id &&
             adam_bind == o.adam_bind && sigma == o.sigma && seed == o.seed && lr == o.lr && a.gt == b.gt &&
             a.out_avg == b.out_avg && a.snapshot == b.snapshot && a.state == b.state && a.records == b.records &&
             a.exp_weight == b.exp_weight && a.show_every == b.show_every && a.backtrack_db == b.backtrack_db;
    }
  };
  GraphKey gkey{};
  cudaGraphExec_t gexec = nullptr;
  // notebook path (dip_forward / dip_backward called once per closure): each is replayed as its own CUDA graph over the
  // plan's fixed staging buffers (zbuf / out_saved / dout); rebuilt when the bound pointers change
  cudaGraphExec_t gfwd = nullptr, gbwd = nullptr;
  cudaStream_t gstream = nullptr;
  cudaEvent_t gev_in = nullptr, gev_out = nullptr;
  // weight-gradient chain runs on a private side stream, forked/joined with events (also inside graph capture)
  cudaStream_t wstream = nullptr;
  // the skip branches (1x1 conv + BN of every level, forward and backward) are independent of the deeper-level chain:
  // they run on a second side stream
  cudaStream_t sstream = nullptr;
  std::vector<cudaEvent_t> wev;
  size_t wev_used = 0;
  bool side_on = false;
  // weight-gradient GEMMs of the outer levels deferred until the main chain is inside the (latency-bound, SM-starved)
  // deep levels, where a full-GPU tensor-core kernel on the side stream costs the least
  std::vector<dip::ConvOp*> deferred;
  // runner: the input perturbation is generated inside the level-0 input transform (k_noise_pad) -- set around plan_forward
  struct { bool on = false; const float* z0 = nullptr; float sigma = 0.f; uint64_t seed = 0, offset = 0; const int* it_dev = nullptr; } fnoise;
  bool prepacked = false;   // the runner already issued the weight repack of this forward (beside the noise kernel)
  // tables
  PackEntry* d_pack = nullptr; CvtEntry* d_cvt = nullptr; RunEntry* d_run = nullptr; UnpackEntry* d_unpack = nullptr;
  int n_pack = 0, n_cvt = 0, n_run = 0, n_unpack = 0;
  float* wacc_base = nullptr; size_t wacc_bytes = 0;   // all weight-gradient accumulators, contiguous
  long long pack_max = 0;
  bool bound = false;
  int nbt_is_float = 0;
  int launches_fwd = 0, launches_bwd = 0;
  Timer timer;
  Recorder rec{&timer};   // plan_forward (with the runner's early repack) and plan_backward
};

namespace dip {

static BnRef bn_ref(const dip_plan* P, const BnLayer& b) {
  BnRef r;
  r.fwd = b.fwd; r.gamma = P->params[b.p_gamma]; r.beta = P->params[b.p_beta];
  r.C = b.C; r.rot = b.rot; r.inv_n = 1.f / b.n;
  return r;
}

static int build_plan(dip_plan* P, Arena& A) {
  const dip_net_desc& d = P->desc;
  const int L = d.num_scales;
  if (L < 1 || L > 8) return fail("dip-b200: 1..8 scales supported");
  // widths: one value for every scale (channels / skip_channels), or per scale (channels == 0: channels_down / channels_up /
  // channels_skip, denoising.ipynb c8:17-23 "snail": [8, 16, 32, 64, 128] with skips [0, 0, 0, 4, 4])
  std::vector<int> ND(L), NU(L), NS(L);
  for (int l = 0; l < L; ++l) {
    ND[l] = d.channels > 0 ? d.channels : d.channels_down[l];
    NU[l] = d.channels > 0 ? d.channels : d.channels_up[l];
    NS[l] = d.channels > 0 ? d.skip_channels : d.channels_skip[l];
    for (int w : {ND[l], NU[l]})
      if (w < 8 || w > 128 || w % 8 != 0)
        return fail("dip-b200: num_channels_down / num_channels_up must be multiples of 8 in [8, 128] (128 in the BASELINE configurations)");
  }
  bool wide = true, uniform = true;
  for (int l = 0; l < L; ++l) {
    wide = wide && NS[l] == 128 && ND[l] == 128 && NU[l] == 128;
    uniform = uniform && ND[l] == 128 && NU[l] == 128 && NS[l] == NS[0];
  }
  for (int l = 0; l < L; ++l)
    if (!(wide || NS[l] == 0 || NS[l] == 4))
      return fail("dip-b200: num_channels_skip must be 0 or 4 per scale, or 128 at every scale of a 128-wide network");
  const int CS = NS[0];   // the uniform skip width where the code below asks for it (wide: 128)
  if (d.downsample_mode != 0 && d.downsample_mode != 1) return fail("dip-b200: downsample_mode must be 'stride' (0) or 'avg' (1)");
  const bool avg = d.downsample_mode == 1;
  // parameters of the skip branch (conv w, b, BN gamma, beta): absent where num_channels_skip[l] = 0
  // (inpainting.ipynb c14:11-16 "vase": models/skip.py:50-53 then adds `deeper` alone, no Concat)
  auto psl = [&](int l) { return NS[l] > 0 ? 4 : 0; };
  // wide: skip branch on the tensor cores, 256-channel concat (all widths 128, all skips 128)
  if (d.in_channels < 1 || d.in_channels > 128) return fail("dip-b200: input depth must be in [1,128]");
  // level-0 activations are stored with the input depth rounded up to a power of two >= 4 (zero channels); the conv
  // weights keep their real depth (TMA zero-fills the missing channels, the 1x1 skip conv reads its rows by element)
  int cin_eng = 4;
  while (cin_eng < d.in_channels) cin_eng *= 2;
  if (d.out_channels < 1 || d.out_channels > 4) return fail("dip-b200: num_output_channels must be <= 4");
  if (P->H % (1 << L) || P->W % (1 << L)) return fail("dip-b200: H and W must be divisible by 2^num_scales");
  if ((P->H >> L) < 2 || (P->W >> L) < 2)
    return fail("dip-b200: H and W must be at least 2 * 2^num_scales (ReflectionPad2d(1) in front of the deepest 3x3 conv needs 2 "
                "pixels per side: torch raises for the reference's network as well)");
  const int prec = d.precision;
  if (prec != DIP_PRECISION_TF32 && prec != DIP_PRECISION_FP32 && prec != DIP_PRECISION_BF16) return fail("dip-b200: unknown precision");
  const bool bf = prec == DIP_PRECISION_BF16;
  P->lv.resize(L);
  int pidx = 0;
  // parameter slots in net.parameters() order: assigned recursively (pre-order part, then post-order part)
  std::vector<int> pre(L), post(L);
  {
    int idx = 0;
    for (int l = 0; l < L; ++l) { pre[l] = idx; idx += 8 + psl(l); }
    for (int l = L - 1; l >= 0; --l) { post[l] = idx; idx += 10; }
    P->p_head_w = idx; P->p_head_b = idx + 1;
    pidx = idx + 2;
  }
  P->numel.assign(pidx, 0);
  P->bns.clear(); P->convs.clear();
  size_t acc_f = 0, acc_b = 0;
  auto bn_init = [&](BnLayer& b, int C, int rot, int n, int pg, int pbias) {
    b.C = C; b.rot = rot; b.n = (float)n; b.p_gamma = pg; b.p_beta = pg + 1; b.p_bias = pbias;
    P->numel[pg] = C; P->numel[pg + 1] = C;
    acc_f += 2 * C; acc_b += 3 * C;
  };
  for (int l = 0; l < L; ++l) {
    Level& v = P->lv[l];
    v.H = P->H >> l; v.W = P->W >> l; v.h = v.H / 2; v.w = v.W / 2;
    v.nd = ND[l]; v.nu = NU[l]; v.ns = NS[l]; v.cu = l == L - 1 ? ND[l] : NU[l + 1];
    const int CS = v.ns, ps = psl(l);   // (shadow the network-wide values inside the level loop)
    v.Cin = l == 0 ? cin_eng : ND[l - 1];
    v.Cin_act = l == 0 ? d.in_channels : ND[l - 1];
    v.bilinear = d.upsample_bilinear < 0 ? (d.upsample_mask >> l) & 1 : (d.upsample_bilinear != 0);
    const int b0 = pre[l], b1 = post[l];
    // skip conv 1x1 Cin -> CS
    if (CS > 0) {
      v.p_skip_w = b0; v.p_skip_b = b0 + 1;
      P->numel[b0] = (long long)CS * v.Cin_act; P->numel[b0 + 1] = CS;
      bn_init(v.bn_s, CS, 0, v.H * v.W, b0 + 2, b0 + 1);
    } else {
      v.p_skip_w = v.p_skip_b = -1;
      v.bn_s = BnLayer{};
    }
    // down1 3x3 s2
    v.d1.N = v.nd; v.d1.C = v.Cin_act; v.d1.k = 3; v.d1.stride = 2; v.d1.p_w = b0 + ps; v.d1.p_b = b0 + ps + 1;
    P->numel[b0 + ps] = (long long)v.nd * v.Cin_act * 9; P->numel[b0 + ps + 1] = v.nd;
    bn_init(v.bn_d1, v.nd, 0, v.h * v.w, b0 + ps + 2, b0 + ps + 1);
    // down2 3x3
    v.d2.N = v.nd; v.d2.C = v.nd; v.d2.k = 3; v.d2.stride = 1; v.d2.p_w = b0 + ps + 4; v.d2.p_b = b0 + ps + 5;
    P->numel[b0 + ps + 4] = (long long)v.nd * v.nd * 9; P->numel[b0 + ps + 5] = v.nd;
    bn_init(v.bn_d2, v.nd, 0, v.h * v.w, b0 + ps + 6, b0 + ps + 5);
    // concat BN (torch channel order [skip | up], engine order [up | skip])
    bn_init(v.bn_cat, v.cu + CS, CS, v.H * v.W, b1 + 0, -1);
    // up 3x3 (cu+CS) -> nu
    v.up.N = v.nu; v.up.C = v.cu + CS; v.up.k = 3; v.up.stride = 1; v.up.rot = CS; v.up.p_w = b1 + 2; v.up.p_b = b1 + 3;
    if (wide) {
      v.up.do_wgrad = false;
      v.sk.C = v.Cin_act; v.sk.k = 1; v.sk.stride = 1; v.sk.p_w = b0; v.sk.p_b = b0 + 1;
      for (ConvOp* h : {&v.up_a, &v.up_b}) {
        h->C = 128; h->Ctot = 128 + CS; h->k = 3; h->stride = 1; h->rot = CS; h->p_w = b1 + 2; h->p_b = b1 + 3;
        h->do_fprop = false; h->dg_ld = 128 + CS;
      }
      v.up_b.coff = 128;
    }
    P->numel[b1 + 2] = (long long)v.nu * (v.cu + CS) * 9; P->numel[b1 + 3] = v.nu;
    bn_init(v.bn_u, v.nu, 0, v.H * v.W, b1 + 4, b1 + 3);
    // 1x1 nu -> nu
    v.c11.N = v.nu; v.c11.C = v.nu; v.c11.k = 1; v.c11.stride = 1; v.c11.p_w = b1 + 6; v.c11.p_b = b1 + 7;
    P->numel[b1 + 6] = (long long)v.nu * v.nu; P->numel[b1 + 7] = v.nu;
    bn_init(v.bn_v, v.nu, 0, v.H * v.W, b1 + 8, b1 + 7);
  }
  const int NH = NU[0];   // depth of the tensor the RGB head reads
  P->numel[P->p_head_w] = (long long)d.out_channels * NH;
  P->numel[P->p_head_b] = d.out_channels;
  // BN order (running-stat table) follows state_dict order: skip, d1, d2, <deeper>, cat, up, 1x1
  {
    std::vector<BnLayer*> a, b;
    for (int l = 0; l < L; ++l) { if (NS[l] > 0) a.push_back(&P->lv[l].bn_s); a.push_back(&P->lv[l].bn_d1); a.push_back(&P->lv[l].bn_d2); }
    for (int l = L - 1; l >= 0; --l) { a.push_back(&P->lv[l].bn_cat); a.push_back(&P->lv[l].bn_u); a.push_back(&P->lv[l].bn_v); }
    P->bns = a;
    for (size_t i = 0; i < P->bns.size(); ++i) P->bns[i]->idx = (int)i;
  }
  // ---- accumulators
  size_t skinny_acc = 0;
  for (int l = 0; l < L; ++l) skinny_acc += (size_t)NS[l] * P->lv[l].Cin;
  skinny_acc += (size_t)d.out_channels * NH + 8;
  P->acc_fwd_n = acc_f * kAccS;
  P->acc_bwd_n = (acc_b + skinny_acc) * kAccS;
  P->acc_fwd = A.get<double>(P->acc_fwd_n);
  P->acc_bwd = A.get<double>(P->acc_bwd_n);
  {
    double* f = P->acc_fwd; double* b = P->acc_bwd;
    for (BnLayer* bn : P->bns) {
      bn->fwd = f; f = f ? f + 2 * bn->C * kAccS : nullptr;
      bn->bwd = b; bn->dbias = b ? b + 2 * bn->C * kAccS : nullptr; b = b ? b + 3 * bn->C * kAccS : nullptr;
    }
    for (int l = 0; l < L; ++l) { P->lv[l].dw_s = b; b = b ? b + (size_t)NS[l] * P->lv[l].Cin * kAccS : nullptr; }
    P->dw_head = b; b = b ? b + (size_t)d.out_channels * NH * kAccS : nullptr;
    P->db_head = b;
    P->db_scratch = b ? b + 4 * kAccS : nullptr;
  }
  // ---- activations.  One statement allocates each level buffer [rows][cols][ld] (c valid channels) and registers it as
  // L<l>.<name> (dip_plan_buffer), under the condition on which a launch of the plan writes it.
  auto reg = [&](const std::string& name, void* p, int rows, int cols, int ld, int c) { P->bufs[name] = BufInfo{p, rows, cols, ld, c}; };
  for (int l = 0; l < L; ++l) {
    Level& v = P->lv[l];
    const std::string pf = "L" + std::to_string(l) + ".";
    auto f32 = [&](const char* name, int rows, int cols, int ld, int c) {
      float* p = A.get<float>((size_t)rows * cols * ld);
      reg(pf + name, p, rows, cols, ld, c);
      return p;
    };
    auto b16 = [&](const char* name, int rows, int cols, int ld, int c) {   // bf16 twin (names end in "16")
      uint16_t* p = A.get<uint16_t>((size_t)rows * cols * ld);
      reg(pf + name, p, rows, cols, ld, c);
      return p;
    };
    const bool last = l == L - 1;
    const int CS = v.ns, nd = v.nd, nu = v.nu, CC = v.cu + v.ns;
    const bool d1_dgrad = l > 0 || d.input_grad != 0;   // level 0 has an input gradient with input_grad only
    if (l == 0) v.Pin = f32("Pin", v.H + 2, v.W + 2, v.Cin, v.Cin);
    else reg(pf + "Pin", v.Pin = P->lv[l - 1].P_d2, v.H + 2, v.W + 2, v.Cin, v.Cin);
    v.raw_s = f32("raw_s", v.H, v.W, CS, CS);
    v.raw_d1 = f32("raw_d1", v.h, v.w, nd, nd);
    v.P_d1 = f32("P_d1", v.h + 2, v.w + 2, nd, nd);
    v.raw_d2 = f32("raw_d2", v.h, v.w, nd, nd);
    v.P_d2 = last ? f32("P_d2", v.h, v.w, nd, nd) : f32("P_d2", v.h + 2, v.w + 2, nd, nd);
    v.P_cat = f32("P_cat", v.H + 2, v.W + 2, CC, CC);
    v.raw_u = f32("raw_u", v.H, v.W, nu, nu);
    v.A_u = f32("A_u", v.H, v.W, nu, nu);
    v.raw_v = f32("raw_v", v.H, v.W, nu, nu);
    v.U = (l > 0 || nu != 128) ? f32("U", v.H, v.W, nu, nu) : nullptr;  // a 128-deep level 0 feeds the fused RGB head instead
    v.dRaw_v = f32("dRaw_v", v.H, v.W, nu, nu);
    v.dA_u = f32("dA_u", v.H, v.W, nu, nu);
    v.dRaw_u = f32("dRaw_u", v.H, v.W, nu, nu);
    v.dP_cat = f32("dP_cat", v.H + 2, v.W + 2, CC, CC);
    v.dCat = f32("dCat", v.H, v.W, CC, CC);
    v.dRaw_s = f32("dRaw_s", v.H, v.W, CS, CS);
    v.dUp = f32("dUp", v.h, v.w, v.cu, v.cu);
    v.dRaw_d2 = f32("dRaw_d2", v.h, v.w, nd, nd);
    v.dP_d1 = f32("dP_d1", v.h + 2, v.w + 2, nd, nd);
    v.dRaw_d1 = f32("dRaw_d1", v.h, v.w, nd, nd);
    if (avg) {
      v.rawF = f32("rawF", v.H, v.W, nd, nd);
      if (bf) v.dRawF16 = b16("dRawF16", v.H, v.W, nd, nd);   // bf16 mode writes the conv's dY as the twin only
      else v.dRawF = f32("dRawF", v.H, v.W, nd, nd);
    }
    // input gradient of the skip conv: the tensor-core 1x1 of skip=128 (levels > 0), or at level 0 the skip conv's part
    // of the network's input gradient
    v.dS = (CS > 0 && (l > 0 ? wide : d.input_grad != 0)) ? f32("dS", v.H, v.W, v.Cin, v.Cin) : nullptr;
    // (level 0: the input gradient conv writes the real input depth only; the stored depth's extra channels are never
    // written, and k_input_grad never reads them)
    v.dPin = d1_dgrad ? f32("dPin", v.H + 2, v.W + 2, v.Cin, v.Cin_act) : nullptr;
    if (bf) {   // bf16 twins of the conv operands (ld = the fp32 tensor's depth rounded up to 8)
      v.Pin_ld16 = round_up(v.Cin, 8); v.cat_ld16 = round_up(CC, 8);
      if (l == 0) v.Pin16 = b16("Pin16", v.H + 2, v.W + 2, v.Pin_ld16, v.Cin);
      else reg(pf + "Pin16", v.Pin16 = P->lv[l - 1].P_d2_16, v.H + 2, v.W + 2, v.Pin_ld16, v.Cin);
      v.P_d1_16 = b16("P_d1_16", v.h + 2, v.w + 2, nd, nd);
      v.P_d2_16 = last ? nullptr : b16("P_d2_16", v.h + 2, v.w + 2, nd, nd);
      v.P_cat16 = b16("P_cat16", v.H + 2, v.W + 2, v.cat_ld16, CC);
      v.A_u16 = b16("A_u16", v.H, v.W, nu, nu);
      v.dRaw_v16 = b16("dRaw_v16", v.H, v.W, nu, nu);
      v.dRaw_u16 = b16("dRaw_u16", v.H, v.W, nu, nu);
      v.dRaw_d2_16 = b16("dRaw_d2_16", v.h, v.w, nd, nd);
      v.dRaw_d1_16 = avg ? nullptr : b16("dRaw_d1_16", v.h, v.w, nd, nd);   // (avg: the pooled gradient stays fp32)
      v.dRaw_s16 = wide ? b16("dRaw_s16", v.H, v.W, 128, 128) : nullptr;
    }
  }
  P->out_saved = A.get<float>((size_t)P->H * P->W * d.out_channels);
  P->zbuf = A.get<float>((size_t)P->H * P->W * d.in_channels);
  P->dout = A.get<float>((size_t)P->H * P->W * d.out_channels);
  P->dl4 = A.get<float>((size_t)P->H * P->W * 4);
  P->ds_kern = A.get<float>(dip_plan::kDownMaxK * dip_plan::kDownMaxK);
  P->ds_y = A.get<float>((size_t)P->H * P->W * d.out_channels);
  P->ds_dy = A.get<float>((size_t)P->H * P->W * d.out_channels);
  P->loss_ring = A.get<double>(dip_plan::kLossRing);
  P->it_dev = A.get<int>(4);
  // ---- conv ops
  size_t partial_max = 0;
  for (int l = 0; l < L; ++l) {
    Level& v = P->lv[l];
    // down1: Pin (padded, stride 2) -> raw_d1
    ConvOp& a = v.d1;
    a.set_shapes();
    a.in = v.Pin; a.in_rows = v.H + 2; a.in_cols = v.W + 2; a.in_ld = v.Cin; a.offx = a.offy = 0;
    a.out = v.raw_d1; a.out_h = v.h; a.out_w = v.w; a.stats = v.bn_d1.fwd;
    a.has_dgrad = l > 0 || d.input_grad != 0;
    a.dg_ld = v.Cin;   // level 0: stored depth (>= the conv's real input depth)
    a.dg_s2 = true;
    a.dy = v.dRaw_d1; a.dy16 = v.dRaw_d1_16;
    a.dg_out = v.dPin; a.dg_out_h = v.H + 2; a.dg_out_w = v.W + 2; a.dg_off = -2;
    a.in16 = v.Pin16; a.in_ld16 = v.Pin_ld16;
    if (avg) {   // stride-1 conv at the level's full resolution; pooling is a separate pass (fwd_level / bwd_level)
      a.stride = 1; a.out = v.rawF; a.out_h = v.H; a.out_w = v.W; a.stats = nullptr;
      a.dg_s2 = false; a.dy = v.dRawF; a.dy16 = v.dRawF16;
    }
    // down2: P_d1 -> raw_d2
    ConvOp& b = v.d2;
    b.set_shapes();
    b.in = v.P_d1; b.in_rows = v.h + 2; b.in_cols = v.w + 2; b.in_ld = v.nd; b.offx = b.offy = 0;
    b.out = v.raw_d2; b.out_h = v.h; b.out_w = v.w; b.stats = v.bn_d2.fwd;
    b.has_dgrad = true;
    b.dy = v.dRaw_d2; b.dy16 = v.dRaw_d2_16;
    b.dg_out = v.dP_d1; b.dg_out_h = v.h + 2; b.dg_out_w = v.w + 2; b.dg_off = -2;
    b.in16 = v.P_d1_16; b.in_ld16 = v.nd;
    // up: P_cat -> raw_u
    ConvOp& c = v.up;
    c.set_shapes();
    c.in = v.P_cat; c.in_rows = v.H + 2; c.in_cols = v.W + 2; c.in_ld = v.cu + v.ns; c.offx = c.offy = 0;
    c.out = v.raw_u; c.out_h = v.H; c.out_w = v.W; c.stats = v.bn_u.fwd;
    c.has_dgrad = !wide;
    c.dy = v.dRaw_u; c.dy16 = v.dRaw_u16;
    c.dg_out = v.dP_cat; c.dg_out_h = v.H + 2; c.dg_out_w = v.W + 2; c.dg_off = -2;
    c.in16 = v.P_cat16; c.in_ld16 = v.cat_ld16;
    // 1x1: A_u -> raw_v
    ConvOp& e = v.c11;
    e.set_shapes();
    e.in = v.A_u; e.in_rows = v.H; e.in_cols = v.W; e.in_ld = v.nu; e.offx = e.offy = 0;
    e.out = v.raw_v; e.out_h = v.H; e.out_w = v.W; e.stats = v.bn_v.fwd;
    e.has_dgrad = true;
    e.dy = v.dRaw_v; e.dy16 = v.dRaw_v16;
    e.dg_out = v.dA_u; e.dg_out_h = v.H; e.dg_out_w = v.W; e.dg_off = 0;
    e.in16 = v.A_u16; e.in_ld16 = v.nu;
    std::vector<ConvOp*> ops = {&a, &b, &c, &e};
    if (wide) {
      // skip conv 1x1 on the interior of the padded level input
      ConvOp& k1 = v.sk;
      k1.set_shapes();
      k1.in = v.Pin; k1.in_rows = v.H + 2; k1.in_cols = v.W + 2; k1.in_ld = v.Cin; k1.offx = k1.offy = 1;
      k1.out = v.raw_s; k1.out_h = v.H; k1.out_w = v.W; k1.stats = v.bn_s.fwd;
      k1.has_dgrad = l > 0 || d.input_grad != 0;
      k1.dg_ld = v.Cin;
      k1.dy = v.dRaw_s; k1.dy16 = v.dRaw_s16;
      k1.dg_out = v.dS; k1.dg_out_h = v.H; k1.dg_out_w = v.W; k1.dg_off = 0;
      k1.in16 = v.Pin16; k1.in_ld16 = v.Pin_ld16;
      ops.push_back(&k1);
      for (ConvOp* h : {&v.up_a, &v.up_b}) {
        h->set_shapes();
        h->in = v.P_cat + h->coff; h->in_rows = v.H + 2; h->in_cols = v.W + 2; h->in_ld = 128 + CS; h->offx = h->offy = 0;
        h->out = v.raw_u; h->out_h = v.H; h->out_w = v.W; h->stats = nullptr;
        h->has_dgrad = true;
        h->dy = v.dRaw_u; h->dy16 = v.dRaw_u16;
        h->dg_out = v.dP_cat + h->coff; h->dg_out_h = v.H + 2; h->dg_out_w = v.W + 2; h->dg_off = -2;
        h->in16 = v.P_cat16 != nullptr ? v.P_cat16 + h->coff : nullptr; h->in_ld16 = v.cat_ld16;
        ops.push_back(h);
      }
    }
    for (ConvOp* op : ops) {
      op->wp_f = op->do_fprop ? A.get<float>(op->wp_f_elems()) : nullptr;
      op->wp_d = op->has_dgrad ? A.get<float>(op->wp_d_elems()) : nullptr;
      op->bf16 = bf;
      op->rec = &P->rec;
      const size_t pe = op->do_wgrad ? op->partial_elems(prec) : 0;
      if (pe > partial_max) partial_max = pe;
      P->convs.push_back(op);
    }
  }
  // split-K partials of the weight gradients.  fp32 mode: one area that every conv's wgrad writes and its own unpack entry
  // sums right away.  Tensor-core modes: every conv's partials in their own slice of one contiguous area, summed by one
  // launch over all entries at the end of the backward pass.
  P->partial = is_tc(prec) ? nullptr : A.get<float>(partial_max);
  P->n_unpack = 0;
  for (ConvOp* op : P->convs) if (op->do_wgrad) P->n_unpack++;
  if (is_tc(prec)) {
    size_t tot = 0;
    for (ConvOp* op : P->convs) if (op->do_wgrad) tot += (op->partial_elems(prec) + 63) & ~size_t(63);
    P->wacc_base = A.get<float>(tot);
    P->wacc_bytes = tot * sizeof(float);
    if (P->wacc_base != nullptr) reg("wacc", P->wacc_base, 1, 1, (int)tot, (int)tot);   // (tests NaN-fill it)
    size_t off = 0;
    for (ConvOp* op : P->convs) if (op->do_wgrad) { op->partial = P->wacc_base ? P->wacc_base + off : nullptr; off += (op->partial_elems(prec) + 63) & ~size_t(63); }
  }
  P->d_unpack = A.get<UnpackEntry>(P->n_unpack > 0 ? P->n_unpack : 1);
  if (!is_tc(prec) && !P->dry) {
    int i = 0;
    for (ConvOp* op : P->convs) if (op->do_wgrad) { op->partial = P->partial; op->unpack = P->d_unpack + i++; }
  }
  P->n_pack = (int)P->convs.size();
  P->n_cvt = (int)P->bns.size() * 3 + L + 2;
  P->n_run = (int)P->bns.size();
  P->d_pack = A.get<PackEntry>(P->n_pack);
  P->d_cvt = A.get<CvtEntry>(P->n_cvt);
  P->d_run = A.get<RunEntry>(P->n_run);
  if (P->dry) return 0;
  // ---- device-side setup
  {
    // side streams at the lowest priority, the graph stream (= main chain of the captured step) at the highest
    int lo = 0, hi = 0;
    DIP_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
    if (getenv("DIP_NO_PRIO") != nullptr) lo = hi = 0;
    DIP_CUDA(cudaStreamCreateWithPriority(&P->wstream, cudaStreamNonBlocking, lo));
    DIP_CUDA(cudaStreamCreateWithPriority(&P->sstream, cudaStreamNonBlocking, lo));
  }
  if (is_tc(prec))
    for (ConvOp* op : P->convs) DIP_CHECK(op->build_tc());
  P->pack_max = 0;
  for (ConvOp* op : P->convs) {
    const long long n = (op->do_fprop ? (long long)op->wp_f_elems() : 0) + (op->has_dgrad ? (long long)op->wp_d_elems() : 0);
    if (n > P->pack_max) P->pack_max = n;
  }
  return 0;
}

static int upload_tables(dip_plan* P) {
  std::vector<PackEntry> pk;
  for (ConvOp* op : P->convs) pk.push_back(op->pack_entry(P->desc.precision, P->params[op->p_w]));
  DIP_CUDA(cudaMemcpy(P->d_pack, pk.data(), pk.size() * sizeof(PackEntry), cudaMemcpyHostToDevice));
  if (P->n_unpack > 0) {
    std::vector<UnpackEntry> up;
    for (ConvOp* op : P->convs)
      if (op->do_wgrad) up.push_back(op->unpack_entry(P->desc.precision, P->grads[op->p_w]));
    if ((int)up.size() != P->n_unpack) return fail("internal: unpack table size mismatch");
    DIP_CUDA(cudaMemcpy(P->d_unpack, up.data(), up.size() * sizeof(UnpackEntry), cudaMemcpyHostToDevice));
  }
  std::vector<CvtEntry> cv;
  for (BnLayer* b : P->bns) {
    cv.push_back(CvtEntry{b->bwd + b->C * kAccS, P->grads[b->p_gamma], b->C, b->rot});  // dgamma = sum dz*xhat
    cv.push_back(CvtEntry{b->bwd, P->grads[b->p_beta], b->C, b->rot});          // dbeta  = sum dz
    if (b->p_bias >= 0) cv.push_back(CvtEntry{b->dbias, P->grads[b->p_bias], b->C, 0});
    else cv.push_back(CvtEntry{b->dbias, nullptr, 0, 0});
  }
  for (size_t l = 0; l < P->lv.size(); ++l) {
    // skip=128: the skip conv's weight gradient comes from the tensor-core wgrad, not from fp64 accumulators
    if (P->lv[l].ns == 128 || P->lv[l].ns == 0) cv.push_back(CvtEntry{P->lv[l].dw_s, nullptr, 0, 0});
    else cv.push_back(CvtEntry{P->lv[l].dw_s, P->grads[P->lv[l].p_skip_w], (int)P->numel[P->lv[l].p_skip_w], 0,
                               P->lv[l].Cin_act, P->lv[l].Cin});   // accumulator rows hold the stored depth
  }
  cv.push_back(CvtEntry{P->dw_head, P->grads[P->p_head_w], (int)P->numel[P->p_head_w], 0});
  cv.push_back(CvtEntry{P->db_head, P->grads[P->p_head_b], (int)P->numel[P->p_head_b], 0});
  if ((int)cv.size() != P->n_cvt) return fail("internal: cvt table size mismatch");
  DIP_CUDA(cudaMemcpy(P->d_cvt, cv.data(), cv.size() * sizeof(CvtEntry), cudaMemcpyHostToDevice));
  std::vector<RunEntry> rn;
  for (BnLayer* b : P->bns) {
    RunEntry e{};
    e.fwd = b->fwd; e.C = b->C; e.rot = b->rot; e.n = b->n;
    if (!P->running.empty()) {
      e.rm = (float*)P->running[3 * b->idx]; e.rv = (float*)P->running[3 * b->idx + 1]; e.nb = P->running[3 * b->idx + 2];
      e.nb_is_float = P->nbt_is_float;
    }
    rn.push_back(e);
  }
  DIP_CUDA(cudaMemcpy(P->d_run, rn.data(), rn.size() * sizeof(RunEntry), cudaMemcpyHostToDevice));
  return 0;
}

// ------------------------------------------------------------------------------------------------ side streams
// Dependency edge between two streams (event record + wait; inside graph capture this becomes a graph edge).
static void stream_edge(dip_plan* P, cudaStream_t from, cudaStream_t to) {
  if (P->wev_used == P->wev.size()) {
    cudaEvent_t e;
    cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
    P->wev.push_back(e);
  }
  cudaEvent_t e = P->wev[P->wev_used++];
  cudaEventRecord(e, from);
  cudaStreamWaitEvent(to, e, 0);
}
// Stream on which the weight-gradient work that depends on everything recorded so far on `s` may run concurrently.
static cudaStream_t fork_side(dip_plan* P, cudaStream_t s) {
  if (!P->side_on) return s;
  stream_edge(P, s, P->wstream);
  return P->wstream;
}
static void join_side(dip_plan* P, cudaStream_t s) {
  if (P->side_on) stream_edge(P, P->wstream, s);
}
// Same for the skip-branch stream.
static bool skip_stream_on(const dip_plan* P) {
  static const bool off = getenv("DIP_NO_SKIPSTREAM") != nullptr;   // experiment switch
  return P->side_on && !off;
}
static cudaStream_t fork_skip(dip_plan* P, cudaStream_t s) {
  if (!skip_stream_on(P)) return s;
  stream_edge(P, s, P->sstream);
  return P->sstream;
}
static void join_skip(dip_plan* P, cudaStream_t s) {
  if (skip_stream_on(P)) stream_edge(P, P->sstream, s);
}

// ------------------------------------------------------------------------------------------------ forward
static CatArgs cat_args(const dip_plan* P, const Level& v, const float* Usrc) {
  CatArgs a;
  a.U = Usrc; a.raw_s = v.raw_s;
  if (v.ns > 0) a.bn_s = bn_ref(P, v.bn_s);
  else a.bn_s = BnRef{nullptr, nullptr, nullptr, 0, 0, 0.f};   // num_channels_skip = 0: the "concat" is the upsampled tensor alone
  a.Cu = v.cu; a.Cs = v.ns; a.H = v.H; a.W = v.W; a.bilinear = v.bilinear;
  return a;
}
static const float* level_usrc(const dip_plan* P, int l) {
  const int L = (int)P->lv.size();
  return l == L - 1 ? P->lv[l].P_d2 : P->lv[l + 1].U;
}

static int fwd_level(dip_plan* P, int l, cudaStream_t s) {
  Level& v = P->lv[l];
  const int prec = P->desc.precision;
  const int CS = v.ns, nd = v.nd, nu = v.nu;
  const bool last = l == (int)P->lv.size() - 1;
  const float* pin_interior = v.Pin + ((size_t)(v.W + 2) + 1) * v.Cin;
  // precision mode bf16: conv inputs are written as bf16 twins; the fp32 tensor is dropped where only convolutions read it
  const bool bf = prec == DIP_PRECISION_BF16;
  // skip branch: 1x1 conv Cin -> CS (+ statistics); independent of the deeper branch until the concat -> skip stream
  if (CS > 0) {
    cudaStream_t ks = fork_skip(P, s);
    if (CS == 128)
      DIP_CHECK(v.sk.run_fprop(prec, P->params[v.p_skip_b], ks));
    else
      ENQ(&P->rec, hbm(H_SKINNY_FWD, 0), (double)v.H * v.W * (v.Cin_act + CS) * sizeof(float), ks,
          launch_skinny_fwd(pin_interior, v.Cin, v.W + 2, P->params[v.p_skip_w], P->params[v.p_skip_b], v.Cin, CS, v.H, v.W, v.raw_s, 0,
                            v.bn_s.fwd, ks, v.Cin_act));
  }
  // deeper branch
  DIP_CHECK(v.d1.run_fprop(prec, P->params[v.d1.p_b], s));
  if (v.rawF != nullptr) {   // downsample_mode 'avg': pool the stride-1 conv output, then the statistics of the pooled tensor
    ENQ(&P->rec, kUntimed, 0, s, launch_avgpool2(v.rawF, v.h, v.w, nd, v.raw_d1, s));
    ENQ(&P->rec, kUntimed, 0, s, launch_channel_stats(v.raw_d1, nd, nd, v.h * v.w, v.bn_d1.fwd, s));
  }
  ENQ(&P->rec, hbm(H_BN_ACT_WRITE, 1), (double)nd * ((double)v.h * v.w + (double)(v.h + 2) * (v.w + 2)) * sizeof(float), s,
      launch_bn_act_write(v.raw_d1, nd, bn_ref(P, v.bn_d1), v.h, v.w, bf ? nullptr : v.P_d1, nd, 1, 1, P->act_fun, s, Twin{v.P_d1_16, nd},
                          P->zero_pad));
  DIP_CHECK(v.d2.run_fprop(prec, P->params[v.d2.p_b], s));
  ENQ(&P->rec, hbm(H_BN_ACT_WRITE, last ? 0 : 1),
      (double)nd * ((double)v.h * v.w + (last ? (double)v.h * v.w : (double)(v.h + 2) * (v.w + 2))) * sizeof(float), s,
      launch_bn_act_write(v.raw_d2, nd, bn_ref(P, v.bn_d2), v.h, v.w, (bf && !last && P->lv[l + 1].ns != 4) ? nullptr : v.P_d2, nd, last ? 0 : 1, 1, P->act_fun, s,
                          Twin{last ? nullptr : v.P_d2_16, nd}, P->zero_pad));   // (the 4-channel skip conv of the next level reads the fp32 tensor)
  if (!last) DIP_CHECK(fwd_level(P, l + 1, s));
  // upsample + concat + BN + pad
  if (CS > 0) join_skip(P, s);
  CatArgs ca = cat_args(P, v, level_usrc(P, l));
  const double cat_in = ((double)v.cu * v.h * v.w + (double)CS * v.H * v.W) * sizeof(float);
  ENQ(&P->rec, hbm(H_CAT_STATS, v.bilinear), cat_in, s, launch_cat_stats(ca, v.bn_cat.fwd, P->act_fun, s));
  ENQ(&P->rec, hbm(H_CAT_WRITE, v.bilinear), cat_in + ((double)v.cu + CS) * (v.H + 2) * (v.W + 2) * sizeof(float), s,
      launch_cat_write(ca, bn_ref(P, v.bn_cat), v.P_cat, P->act_fun, s, Twin{v.P_cat16, v.cat_ld16}, P->zero_pad));
  DIP_CHECK(v.up.run_fprop(prec, P->params[v.up.p_b], s));
  ENQ(&P->rec, hbm(H_BN_ACT_WRITE, 0), 2.0 * nu * v.H * v.W * sizeof(float), s,
      launch_bn_act_write(v.raw_u, nu, bn_ref(P, v.bn_u), v.H, v.W, bf ? nullptr : v.A_u, nu, 0, 1, P->act_fun, s, Twin{v.A_u16, nu}));
  DIP_CHECK(v.c11.run_fprop(prec, P->params[v.c11.p_b], s));
  if (l > 0 || nu != 128) {
    ENQ(&P->rec, hbm(H_BN_ACT_WRITE, 0), 2.0 * nu * v.H * v.W * sizeof(float), s,
        launch_bn_act_write(v.raw_v, nu, bn_ref(P, v.bn_v), v.H, v.W, v.U, nu, 0, 1, P->act_fun, s));
    if (l == 0) {
      // level 0 narrower than 128 channels: the RGB head (models/skip.py:95-98) as a skinny 1x1 conv over the materialised
      // activation (the fused BN + head kernel is specialised for 128 channels = one warp per pixel)
      ENQ(&P->rec, hbm(H_SKINNY_FWD, 1), ((double)nu + P->desc.out_channels) * v.H * v.W * sizeof(float), s,
          launch_skinny_fwd(v.U, nu, v.W, P->params[P->p_head_w], P->params[P->p_head_b], nu, P->desc.out_channels, v.H, v.W,
                            P->out_saved, P->desc.need_sigmoid != 0 ? 1 : 2, nullptr, s));
    }
  } else {
    // top level: BN + activation + RGB head + sigmoid in one pass; the 128-channel activation is never materialised
    HeadRef hd{P->params[P->p_head_w], P->params[P->p_head_b], P->desc.out_channels, P->out_saved, P->desc.need_sigmoid != 0};
    ENQ(&P->rec, hbm(H_BN_ACT_HEAD, 0), (128.0 + P->desc.out_channels) * v.H * v.W * sizeof(float), s,
        launch_bn_act_head(v.raw_v, bn_ref(P, v.bn_v), v.H, v.W, hd, P->act_fun, s));
  }
  DIP_CUDA(cudaGetLastError());
  return 0;
}

// one table-driven launch repacks the weights of all wide convs (OIHW -> per-tap K-major fprop / dgrad operands)
static void plan_pack(dip_plan* P, cudaStream_t s) {
  dim3 grid((unsigned)((P->pack_max + 255) / 256 < 64 ? (P->pack_max + 255) / 256 : 64), P->n_pack);
  double bytes = 0;
  for (ConvOp* op : P->convs)
    bytes += ((double)op->N * op->C * op->k * op->k + (op->do_fprop ? (double)op->wp_f_elems() : 0.0) + (op->has_dgrad ? (double)op->wp_d_elems() : 0.0)) * sizeof(float);
  ENQ(&P->rec, hbm(H_PACK, 0), bytes, s, launch_k(k_pack_table, dim3(grid), dim3(256), 0, s, 1, P->d_pack));
}

static int plan_forward(dip_plan* P, const float* z, const float* noise, float sigma, float* out, cudaStream_t s) {
  if (!P->bound) return fail("dip_forward: parameters not bound (call dip_plan_bind)");
  // grid-wide reductions: fp64 atomics onto line-strided accumulators (default) or the deterministic last-block sum
  P->side_on = getenv("DIP_NO_SIDE") == nullptr;
  if (!P->prepacked) { P->wev_used = 0; P->rec.n = 0; }
  ENQ(&P->rec, kUntimed, 0, s, DIP_CUDA(cudaMemsetAsync(P->acc_fwd, 0, P->acc_fwd_n * sizeof(double), s)));
  if (!P->prepacked) plan_pack(P, fork_side(P, s));   // weight repack runs beside the input transform
  P->prepacked = false;
  Level& v0 = P->lv[0];
  if (P->fnoise.on)
    ENQ(&P->rec, hbm(H_NOISE, 1), ((double)v0.Cin_act * v0.H * v0.W + (double)v0.Cin * (v0.H + 2) * (v0.W + 2)) * sizeof(float), s,
        launch_noise_pad(P->fnoise.z0, P->fnoise.sigma, P->fnoise.seed, P->fnoise.offset, P->fnoise.it_dev, v0.Pin, v0.Cin,
                         v0.H, v0.W, v0.Cin_act, s, Twin{v0.Pin16, v0.Pin_ld16}, P->zero_pad));
  else
    ENQ(&P->rec, hbm(H_INPUT_PAD, noise != nullptr),
        ((noise != nullptr ? 2.0 : 1.0) * v0.Cin_act * v0.H * v0.W + (double)v0.Cin * (v0.H + 2) * (v0.W + 2)) * sizeof(float), s,
        launch_input_pad(z, noise, sigma, v0.Pin, v0.Cin, v0.H, v0.W, s, v0.Cin_act, Twin{v0.Pin16, v0.Pin_ld16}, P->zero_pad));
  join_side(P, s);
  DIP_CHECK(fwd_level(P, 0, s));
  if (out != nullptr && out != P->out_saved)
    ENQ(&P->rec, kUntimed, 0, s,
        DIP_CUDA(cudaMemcpyAsync(out, P->out_saved, (size_t)v0.H * v0.W * P->desc.out_channels * sizeof(float), cudaMemcpyDeviceToDevice, s)));
  ENQ(&P->rec, kUntimed, 0, s, launch_k(k_running_table, dim3(P->n_run), dim3(160), 0, s, 1, P->d_run));
  DIP_CUDA(cudaGetLastError());
  P->launches_fwd = P->rec.n;
  return 0;
}

// ------------------------------------------------------------------------------------------------ backward
static int bn_bwd(dip_plan* P, const float* raw, int ld_raw, BnLayer& b, int act, GradSrc src, int H, int W, float* draw,
                  cudaStream_t s, uint16_t* draw16 = nullptr) {
  if (draw16 != nullptr) draw = nullptr;   // bf16 mode: only the tensor-core dgrad / wgrad read this gradient
  if (src.kind == 1) src.zero_pad = P->zero_pad;            // zero padding: the padded gradient's halo is dropped, not folded
  BnRef r = bn_ref(P, b);
  // algorithmic bytes: raw + the gradient source as the kernel's contract names it (plain [H][W][C]; fold: the padded
  // dgrad output (+ the 4-channel skip-branch gradient / the plain addend); upsample adjoint: the 2H x 2W gradient; head:
  // the 4 logit gradients per pixel), + the written input gradient for the apply pass
  const double px = (double)H * W, C4 = b.C * sizeof(float);
  double gsrc = px * C4;
  if (src.kind == 1) gsrc = (src.zero_pad ? px : (double)(H + 2) * (W + 2)) * C4 + (src.ds != nullptr ? px * 4 * sizeof(float) : 0.0) + (src.add != nullptr ? px * C4 : 0.0);
  else if (src.kind == 2) gsrc = 4.0 * px * C4;
  else if (src.kind == 3) gsrc = px * 4 * sizeof(float);
  ENQ(&P->rec, hbm(H_BN_BWD_REDUCE, src.kind), px * C4 + gsrc, s, launch_bn_bwd_reduce(raw, ld_raw, r, act, P->act_fun, src, H, W, b.bwd, s));
  ENQ(&P->rec, hbm(H_BN_BWD_APPLY, src.kind), px * C4 + gsrc + px * C4, s,
      launch_bn_bwd_apply(raw, ld_raw, r, act, P->act_fun, src, H, W, b.bwd, draw, b.dbias, s, Twin{draw16, b.C}));
  return 0;
}
static GradSrc src_plain(const float* g, int ld, int coff) { GradSrc s{}; s.kind = 0; s.g = g; s.ld = ld; s.coff = coff; return s; }
// fold of a padded dgrad output; optionally + the dgrad of the next level's 1x1 skip conv computed on the fly
static GradSrc src_fold(const float* gp, int ld, const float* ds, const float* w2, int n2) {
  GradSrc s{}; s.kind = 1; s.g = gp; s.ld = ld; s.coff = 0; s.ds = ds; s.w2 = w2; s.n2 = n2; return s;
}
static GradSrc src_upadj(const float* d, int ld, int bilinear) { GradSrc s{}; s.kind = 2; s.g = d; s.ld = ld; s.coff = 0; s.bilinear = bilinear; return s; }

// Weight gradients of the levels above kDeferLevel are deferred until the backward pass reaches it, so that they run
// beside the deeper levels' launches.
static constexpr int kDeferLevel = 2;
static int flush_deferred(dip_plan* P, int prec, cudaStream_t s) {
  if (P->deferred.empty()) return 0;
  cudaStream_t ws = fork_side(P, s);
  for (ConvOp* op : P->deferred) DIP_CHECK(op->run_wgrad(prec, ws));
  P->deferred.clear();
  return 0;
}
// Weight gradient (side stream) and input gradient (main stream, on the critical path) of one conv.  Both are persistent
// kernels that fill every SM, so they run one after the other whichever way: the dgrad is enqueued first and the main
// stream has the higher priority, so that the wgrad overlaps the HBM-bound kernels that follow the dgrad instead of
// delaying it.
static int conv_backward(dip_plan* P, ConvOp& op, bool dgrad, int prec, cudaStream_t s, int level = 99) {
  if (P->side_on && level < kDeferLevel && (int)P->lv.size() > kDeferLevel) {
    if (dgrad) DIP_CHECK(op.run_dgrad(prec, s));
    P->deferred.push_back(&op);
    return 0;
  }
  cudaStream_t ws = fork_side(P, s);
  if (dgrad) DIP_CHECK(op.run_dgrad(prec, s));
  return op.run_wgrad(prec, ws);
}

static int bwd_level(dip_plan* P, int l, GradSrc src_v, cudaStream_t s) {
  Level& v = P->lv[l];
  const int prec = P->desc.precision;
  const int CS = v.ns, nd = v.nd, nu = v.nu;
  const int CC = v.cu + CS;
  const bool last = l == (int)P->lv.size() - 1;
  // 1x1 conv + BN + LReLU
  DIP_CHECK(bn_bwd(P, v.raw_v, nu, v.bn_v, 1, src_v, v.H, v.W, v.dRaw_v, s, v.dRaw_v16));
  if (l == kDeferLevel) DIP_CHECK(flush_deferred(P, prec, s));
  DIP_CHECK(conv_backward(P, v.c11, true, prec, s, l));
  // up conv + BN + LReLU
  DIP_CHECK(bn_bwd(P, v.raw_u, nu, v.bn_u, 1, src_plain(v.dA_u, nu, 0), v.H, v.W, v.dRaw_u, s, v.dRaw_u16));
  if (CS == 128) {
    cudaStream_t ws = fork_side(P, s);
    DIP_CHECK(v.up_a.run_dgrad(prec, s));
    DIP_CHECK(v.up_b.run_dgrad(prec, s));
    DIP_CHECK(v.up_a.run_wgrad(prec, ws));
    DIP_CHECK(v.up_b.run_wgrad(prec, ws));
  } else {
    DIP_CHECK(conv_backward(P, v.up, true, prec, s, l));
  }
  // concat BN
  BnRef rc = bn_ref(P, v.bn_cat);
  // stored BN output + padded gradient (zero padding: its interior only)
  const double catb = ((double)v.H * v.W + (P->zero_pad ? (double)v.H * v.W : (double)(v.H + 2) * (v.W + 2))) * CC * sizeof(float);
  ENQ(&P->rec, hbm(H_CAT_BWD_REDUCE, 0), catb, s, launch_cat_bwd_reduce(v.P_cat, rc, v.dP_cat, CC, v.H, v.W, v.bn_cat.bwd, s, P->zero_pad));
  ENQ(&P->rec, hbm(H_CAT_BWD_APPLY, 0), catb + (double)v.H * v.W * CC * sizeof(float), s,
      launch_cat_bwd_apply(v.P_cat, rc, v.dP_cat, CC, v.H, v.W, v.bn_cat.bwd, v.dCat, s, P->zero_pad));
  // skip branch (on the skip stream: independent of the deeper levels; the level above joins before it reads dRaw_s / dS)
  cudaStream_t ks = fork_skip(P, s);
  // gradient w.r.t. the low-resolution tensor that was upsampled into this concat (adjoint of x2 upsampling), once
  ENQ(&P->rec, hbm(H_UPADJ, v.bilinear), (double)v.cu * ((double)v.H * v.W + (double)v.h * v.w) * sizeof(float), s,
      launch_upadj(v.dCat, CC, 0, v.h, v.w, v.cu, v.bilinear, v.dUp, s));
  if (CS > 0) DIP_CHECK(bn_bwd(P, v.raw_s, CS, v.bn_s, 1, src_plain(v.dCat, CC, v.cu), v.H, v.W, v.dRaw_s, ks, v.dRaw_s16));
  if (CS == 0) {
    // no skip branch (models/skip.py:50-53 with num_channels_skip = 0)
  } else if (CS == 128) {
    DIP_CHECK(v.sk.run_wgrad(prec, fork_side(P, ks)));
    if (l > 0 || P->desc.input_grad) DIP_CHECK(v.sk.run_dgrad(prec, ks));   // dS, added to the fold of dPin by the level above
  } else {
    const float* pin_interior = v.Pin + ((size_t)(v.W + 2) + 1) * v.Cin;
    // weight gradient only: the input gradient of this conv is folded into the BN backward of the level above
    ENQ(&P->rec, hbm(H_SKINNY_BWD, 0), (double)v.H * v.W * (v.Cin_act + CS) * sizeof(float), ks,
        launch_skinny_bwd(pin_interior, v.Cin, v.W + 2, P->params[v.p_skip_w], v.Cin, CS, v.H, v.W, v.dRaw_s, nullptr, 0,
                          (l == 0 && P->desc.input_grad) ? v.dS : nullptr, v.dw_s, nullptr /*bias grad comes from the BN backward*/, ks, v.Cin_act));
  }
  // deeper branch
  GradSrc src_d2;
  if (!last) {
    DIP_CHECK(bwd_level(P, l + 1, src_plain(v.dUp, v.cu, 0), s));
    join_skip(P, s);   // the next level's skip-branch gradients (dRaw_s / dS) feed the BN backward below
    Level& n = P->lv[l + 1];   // (its input depth n.Cin == nd)
    if (n.ns == 128) { src_d2 = src_fold(n.dPin, nd, nullptr, nullptr, 0); src_d2.add = n.dS; src_d2.ld_add = nd; }
    else if (n.ns == 0) src_d2 = src_fold(n.dPin, nd, nullptr, nullptr, 0);
    else src_d2 = src_fold(n.dPin, nd, n.dRaw_s, P->params[n.p_skip_w], n.ns);
  } else {
    src_d2 = src_plain(v.dUp, v.cu, 0);
  }
  DIP_CHECK(bn_bwd(P, v.raw_d2, nd, v.bn_d2, 1, src_d2, v.h, v.w, v.dRaw_d2, s, v.dRaw_d2_16));
  DIP_CHECK(conv_backward(P, v.d2, true, prec, s));
  const bool d1_dgrad = l > 0 || P->desc.input_grad != 0;
  const bool avg = v.rawF != nullptr;
  DIP_CHECK(bn_bwd(P, v.raw_d1, nd, v.bn_d1, 1, src_fold(v.dP_d1, nd, nullptr, nullptr, 0), v.h, v.w, v.dRaw_d1, s,
                   avg ? nullptr : v.dRaw_d1_16));
  if (avg)   // adjoint of AvgPool2d(2, 2): the conv's dY at full resolution
    ENQ(&P->rec, kUntimed, 0, s,
        launch_avgpool2_bwd(v.dRaw_d1, v.h, v.w, nd, prec == DIP_PRECISION_BF16 ? nullptr : v.dRawF, s, Twin{v.dRawF16, nd}));
  DIP_CHECK(conv_backward(P, v.d1, d1_dgrad, prec, s));
  DIP_CUDA(cudaGetLastError());
  return 0;
}

static int plan_backward(dip_plan* P, const float* dout, cudaStream_t s) {
  if (!P->bound) return fail("dip_backward: parameters not bound");
  P->rec.n = 0;
  P->deferred.clear();
  ENQ(&P->rec, kUntimed, 0, s, DIP_CUDA(cudaMemsetAsync(P->acc_bwd, 0, P->acc_bwd_n * sizeof(double), s)));
  P->side_on = getenv("DIP_NO_SIDE") == nullptr;
  Level& v0 = P->lv[0];
  // RGB head backward (sigmoid', dgrad 3->128, wgrad, bias grad) is fused into the BN backward of the last stage
  GradSrc sh{};
  ENQ(&P->rec, hbm(H_HEAD_DLOGIT, 0), (2.0 * P->desc.out_channels + 4.0) * P->H * P->W * sizeof(float), s,
      launch_head_dlogit(dout, P->out_saved, P->desc.out_channels, P->H * P->W, P->dl4, s, P->desc.need_sigmoid != 0));
  sh.kind = 3; sh.dl4 = P->dl4; sh.wh = P->params[P->p_head_w]; sh.nh = P->desc.out_channels;
  sh.dwh = P->dw_head; sh.dbh = P->db_head;
  DIP_CHECK(bwd_level(P, 0, sh, s));
  DIP_CHECK(flush_deferred(P, P->desc.precision, s));
  join_side(P, s);
  join_skip(P, s);
  ENQ(&P->rec, kUntimed, 0, s, launch_k(k_cvt_table, dim3(P->n_cvt), dim3(128), 0, s, 1, P->d_cvt));
  if (is_tc(P->desc.precision) && P->n_unpack > 0)   // (fp32 mode: each conv's entry ran after its wgrad)
    ENQ(&P->rec, hbm(H_WGRAD_REDUCE, 1), 2.0 * (double)P->wacc_bytes, s,
        launch_k(k_wgrad_unpack_table, dim3(64, P->n_unpack), dim3(256), 0, s, 1, P->d_unpack));
  DIP_CUDA(cudaGetLastError());
  P->launches_bwd = P->rec.n;
  return 0;
}

}  // namespace dip

// ================================================================================================ C ABI
struct dip_adam {
  int n = 0;
  std::vector<long long> numel;
  int nblocks = 0;
  float** d_p = nullptr; const float** d_g = nullptr; float** d_m = nullptr; float** d_v = nullptr;
  int* d_blk_tensor = nullptr; int* d_blk_start = nullptr; int* d_numel = nullptr;
  long long* d_off = nullptr;       // prefix sums of numel: tensor i's offset in a flat buffer (the tracker's snapshot)
  bool bound = false;
  unsigned long long id = 0;        // unique per dip_adam_create (graph cache key of dip_run_iterations)
  unsigned long long bind_gen = 0;  // bumped by dip_adam_bind (the captured k_adam reads the tables, not their addresses,
                                    // but a re-bind after capture must still invalidate nothing else; kept for clarity)
};
static unsigned long long g_adam_serial = 0;

static void drop_graphs(dip_plan* P) {
  for (cudaGraphExec_t* g : {&P->gexec, &P->gfwd, &P->gbwd})
    if (*g != nullptr) { cudaGraphExecDestroy(*g); *g = nullptr; }
}
static bool graphs_enabled(const dip_plan* P) { return !P->timer.on && getenv("DIP_NO_GRAPH") == nullptr; }
static int ensure_gstream(dip_plan* P) {
  // the legacy default stream cannot be captured: graphs replay on a private stream, ordered against the caller's stream
  if (P->gstream == nullptr) {
    int lo = 0, hi = 0;
    DIP_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
    if (getenv("DIP_NO_PRIO") != nullptr) hi = 0;
    DIP_CUDA(cudaStreamCreateWithPriority(&P->gstream, cudaStreamNonBlocking, hi));
    DIP_CUDA(cudaEventCreateWithFlags(&P->gev_in, cudaEventDisableTiming));
    DIP_CUDA(cudaEventCreateWithFlags(&P->gev_out, cudaEventDisableTiming));
  }
  return 0;
}
// Captures body(gs) into *exec (nullptr on failure).
template <class Body>
static int capture_graph(cudaStream_t gs, cudaGraphExec_t* exec, Body body) {
  cudaGraph_t graph = nullptr;
  DIP_CUDA(cudaStreamBeginCapture(gs, cudaStreamCaptureModeThreadLocal));
  const int rc = body(gs);
  cudaError_t ce = cudaStreamEndCapture(gs, &graph);
  if (rc != 0) { if (graph) cudaGraphDestroy(graph); return rc; }
  if (ce != cudaSuccess) return fail(std::string("cudaStreamEndCapture: ") + cudaGetErrorString(ce));
  ce = cudaGraphInstantiate(exec, graph, 0);
  cudaGraphDestroy(graph);
  if (ce != cudaSuccess) { *exec = nullptr; return fail(std::string("cudaGraphInstantiate: ") + cudaGetErrorString(ce)); }
  return 0;
}
// Captures body(gstream) once into *exec, then replays it between two event edges to / from the caller's stream `s`.
template <class Body>
static int replay_graph(dip_plan* P, cudaGraphExec_t* exec, cudaStream_t s, Body body) {
  DIP_CHECK(ensure_gstream(P));
  cudaStream_t gs = P->gstream;
  DIP_CUDA(cudaEventRecord(P->gev_in, s));
  DIP_CUDA(cudaStreamWaitEvent(gs, P->gev_in, 0));
  if (*exec == nullptr) DIP_CHECK(capture_graph(gs, exec, body));
  DIP_CUDA(cudaGraphLaunch(*exec, gs));
  DIP_CUDA(cudaEventRecord(P->gev_out, gs));
  DIP_CUDA(cudaStreamWaitEvent(s, P->gev_out, 0));
  return 0;
}

extern "C" {

const char* dip_last_error(void) { return g_err.c_str(); }
int dip_version(void) { return 100; }

static_assert(DIP_ACT_LEAKY_RELU == kActLeakyRelu && DIP_ACT_SWISH == kActSwish && DIP_ACT_ELU == kActElu &&
                  DIP_ACT_NONE == kActNone, "the plan's act_fun is passed to the kernels as their kAct* kind");
// options -> plan fields; NULL = defaults (reflection padding, LeakyReLU)
static int apply_opts(dip_plan* P, const dip_plan_opts* opts) {
  const int pad = opts != nullptr ? opts->pad_mode : DIP_PAD_REFLECTION;
  if (pad != DIP_PAD_REFLECTION && pad != DIP_PAD_ZERO)
    return fail("dip-b200: pad_mode must be DIP_PAD_REFLECTION (0) or DIP_PAD_ZERO (1), got " + std::to_string(pad));
  const int act = opts != nullptr ? opts->act_fun : DIP_ACT_LEAKY_RELU;
  if (act < DIP_ACT_LEAKY_RELU || act > DIP_ACT_NONE)
    return fail("dip-b200: act_fun must be DIP_ACT_LEAKY_RELU (0), DIP_ACT_SWISH (1), DIP_ACT_ELU (2) or DIP_ACT_NONE (3), got " +
                std::to_string(act));
  P->zero_pad = pad == DIP_PAD_ZERO;
  P->act_fun = act;
  return 0;
}

size_t dip_plan_workspace_bytes_opts(const dip_net_desc* desc, int H, int W, const dip_plan_opts* opts) {
  dip_plan P;
  P.desc = *desc; P.H = H; P.W = W; P.dry = true;
  if (apply_opts(&P, opts) != 0) return 0;
  Arena A{nullptr};
  if (build_plan(&P, A) != 0) return 0;
  return A.off + 4096;
}
size_t dip_plan_workspace_bytes(const dip_net_desc* desc, int H, int W) { return dip_plan_workspace_bytes_opts(desc, H, W, nullptr); }

int dip_plan_create_opts(const dip_net_desc* desc, int H, int W, const dip_plan_opts* opts, void* workspace,
                         size_t workspace_bytes, dip_plan** out) {
  DIP_CHECK(engine_init());
  const size_t need = dip_plan_workspace_bytes_opts(desc, H, W, opts);
  if (need == 0) return -1;
  if (workspace == nullptr || workspace_bytes < need) return fail("dip_plan_create: workspace too small");
  if (reinterpret_cast<uintptr_t>(workspace) % 256 != 0) return fail("dip_plan_create: workspace must be 256-byte aligned");
  dip_plan* P = new dip_plan();
  P->desc = *desc; P->H = H; P->W = W; P->ws = (uint8_t*)workspace; P->ws_bytes = workspace_bytes;
  apply_opts(P, opts);
  Arena A{(uint8_t*)workspace};
  if (build_plan(P, A) != 0) { delete P; return -1; }
  *out = P;
  return 0;
}
int dip_plan_create(const dip_net_desc* desc, int H, int W, void* workspace, size_t workspace_bytes, dip_plan** out) {
  return dip_plan_create_opts(desc, H, W, nullptr, workspace, workspace_bytes, out);
}
void dip_plan_destroy(dip_plan* plan) {
  if (plan == nullptr) return;
  if (plan->gexec) cudaGraphExecDestroy(plan->gexec);
  if (plan->gfwd) cudaGraphExecDestroy(plan->gfwd);
  if (plan->gbwd) cudaGraphExecDestroy(plan->gbwd);
  if (plan->gstream) cudaStreamDestroy(plan->gstream);
  if (plan->gev_in) cudaEventDestroy(plan->gev_in);
  if (plan->gev_out) cudaEventDestroy(plan->gev_out);
  for (cudaEvent_t e : plan->timer.pool) cudaEventDestroy(e);
  for (cudaEvent_t e : plan->wev) cudaEventDestroy(e);
  if (plan->wstream) cudaStreamDestroy(plan->wstream);
  if (plan->sstream) cudaStreamDestroy(plan->sstream);
  delete plan;
}
int dip_plan_num_params(const dip_plan* plan) { return (int)plan->numel.size(); }
int dip_plan_num_bn(const dip_plan* plan) { return (int)plan->bns.size(); }
long long dip_plan_param_numel(const dip_plan* plan, int index) {
  if (index < 0 || index >= (int)plan->numel.size()) return -1;
  return plan->numel[index];
}
int dip_plan_bind(dip_plan* P, void* const* params, void* const* grads, void* const* bn_running, int nbt_is_float) {
  drop_graphs(P);   // captured launches hold the old pointers
  P->nbt_is_float = nbt_is_float;
  const int n = (int)P->numel.size();
  P->params.resize(n); P->grads.resize(n);
  for (int i = 0; i < n; ++i) {
    if (params[i] == nullptr || grads[i] == nullptr) return fail("dip_plan_bind: null parameter/gradient pointer");
    P->params[i] = (float*)params[i]; P->grads[i] = (float*)grads[i];
  }
  P->running.clear();
  if (bn_running != nullptr) P->running.assign(bn_running, bn_running + 3 * P->bns.size());
  DIP_CHECK(upload_tables(P));
  P->bound = true;
  return 0;
}
int dip_forward(dip_plan* P, const void* z, const void* noise, float sigma, void* out, dip_stream_t stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (!P->bound) return fail("dip_forward: parameters not bound (call dip_plan_bind)");
  if (noise != nullptr || !graphs_enabled(P))
    return plan_forward(P, (const float*)z, (const float*)noise, sigma, (float*)out, s);
  // stage the input in the plan's fixed buffer, replay the captured forward, hand the result out
  const size_t nz = (size_t)P->H * P->W * P->desc.in_channels * sizeof(float);
  DIP_CUDA(cudaMemcpyAsync(P->zbuf, z, nz, cudaMemcpyDeviceToDevice, s));
  DIP_CHECK(replay_graph(P, &P->gfwd, s, [&](cudaStream_t gs) { return plan_forward(P, P->zbuf, nullptr, 0.f, nullptr, gs); }));
  if (out != nullptr && out != P->out_saved)
    DIP_CUDA(cudaMemcpyAsync(out, P->out_saved, (size_t)P->H * P->W * P->desc.out_channels * sizeof(float), cudaMemcpyDeviceToDevice, s));
  return 0;
}
int dip_backward(dip_plan* P, const void* dout, dip_stream_t stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (!P->bound) return fail("dip_backward: parameters not bound");
  if (!graphs_enabled(P)) return plan_backward(P, (const float*)dout, s);
  if (dout != P->dout)
    DIP_CUDA(cudaMemcpyAsync(P->dout, dout, (size_t)P->H * P->W * P->desc.out_channels * sizeof(float), cudaMemcpyDeviceToDevice, s));
  return replay_graph(P, &P->gbwd, s, [&](cudaStream_t gs) { return plan_backward(P, P->dout, gs); });
}
int dip_loss_mse(const void* out, const void* target, const void* mask, int channels, int hw, double* loss, void* dout,
                 dip_stream_t stream) {
  launch_mse((const float*)out, (const float*)target, (const float*)mask, channels, hw, loss, (float*)dout, nullptr, (cudaStream_t)stream);
  DIP_CUDA(cudaGetLastError());
  return 0;
}
int dip_noise_perturb(const void* z0, void* z, float sigma, uint64_t seed, uint64_t offset, size_t n, dip_stream_t stream) {
  if (n % 4 != 0) return fail("dip_noise_perturb: n must be a multiple of 4");
  launch_noise((const float*)z0, (float*)z, sigma, seed, offset, nullptr, n, (cudaStream_t)stream);
  DIP_CUDA(cudaGetLastError());
  return 0;
}

int dip_lanczos_down_fwd(const void* x, int C, int H, int W, const void* kern, int K, int factor, int pad, void* y,
                         dip_stream_t stream) {
  DIP_CHECK(engine_init());
  if (K < 1 || factor < 1 || pad < 0) return fail("dip_lanczos_down_fwd: bad K / factor / pad");
  if (down_out_size(H, K, factor, pad) < 1 || down_out_size(W, K, factor, pad) < 1)
    return fail("dip_lanczos_down_fwd: image smaller than the filter");
  DIP_CUDA(launch_down_fwd((const float*)x, C, H, W, (const float*)kern, K, factor, pad, (float*)y, (cudaStream_t)stream));
  return 0;
}
int dip_lanczos_down_bwd(const void* dy, int C, int H, int W, const void* kern, int K, int factor, int pad, void* dx,
                         dip_stream_t stream) {
  DIP_CHECK(engine_init());
  if (K < 1 || factor < 1 || pad < 0) return fail("dip_lanczos_down_bwd: bad K / factor / pad");
  if (down_out_size(H, K, factor, pad) < 1 || down_out_size(W, K, factor, pad) < 1)
    return fail("dip_lanczos_down_bwd: image smaller than the filter");
  DIP_CUDA(launch_down_bwd((const float*)dy, C, H, W, (const float*)kern, K, factor, pad, (float*)dx, (cudaStream_t)stream));
  return 0;
}
int dip_lanczos_down_out_size(int n, int K, int factor, int pad) { return down_out_size(n, K, factor, pad); }

int dip_plan_set_downsampler(dip_plan* P, const float* kern_host, int K, int factor, int pad) {
  if (P->gexec != nullptr) { cudaGraphExecDestroy(P->gexec); P->gexec = nullptr; }   // the captured step changes
  if (kern_host == nullptr || K == 0) { P->ds_K = 0; return 0; }
  if (K < 1 || K > dip_plan::kDownMaxK || factor < 1 || pad < 0) return fail("dip_plan_set_downsampler: bad K / factor / pad");
  const int Ho = down_out_size(P->H, K, factor, pad), Wo = down_out_size(P->W, K, factor, pad);
  if (Ho < 1 || Wo < 1 || Ho > P->H || Wo > P->W) return fail("dip_plan_set_downsampler: unsupported output size");
  DIP_CUDA(cudaMemcpy(P->ds_kern, kern_host, (size_t)K * K * sizeof(float), cudaMemcpyHostToDevice));
  P->ds_K = K; P->ds_f = factor; P->ds_pad = pad; P->ds_Ho = Ho; P->ds_Wo = Wo;
  return 0;
}

int dip_adam_create(int ntensors, const long long* numel, dip_adam** out) {
  dip_adam* a = new dip_adam();
  a->id = ++g_adam_serial;
  a->n = ntensors;
  a->numel.assign(numel, numel + ntensors);
  std::vector<int> bt, bs, ne;
  std::vector<long long> off;
  const int chunk = adam_chunk();
  for (int t = 0; t < ntensors; ++t) {
    off.push_back(t == 0 ? 0 : off.back() + numel[t - 1]);
    ne.push_back((int)numel[t]);
    for (long long st = 0; st < numel[t]; st += chunk) { bt.push_back(t); bs.push_back((int)st); }
  }
  a->nblocks = (int)bt.size();
  DIP_CUDA(cudaMalloc(&a->d_p, ntensors * sizeof(void*)));
  DIP_CUDA(cudaMalloc(&a->d_g, ntensors * sizeof(void*)));
  DIP_CUDA(cudaMalloc(&a->d_m, ntensors * sizeof(void*)));
  DIP_CUDA(cudaMalloc(&a->d_v, ntensors * sizeof(void*)));
  DIP_CUDA(cudaMalloc(&a->d_blk_tensor, bt.size() * sizeof(int)));
  DIP_CUDA(cudaMalloc(&a->d_blk_start, bs.size() * sizeof(int)));
  DIP_CUDA(cudaMalloc(&a->d_numel, ne.size() * sizeof(int)));
  DIP_CUDA(cudaMalloc(&a->d_off, off.size() * sizeof(long long)));
  DIP_CUDA(cudaMemcpy(a->d_blk_tensor, bt.data(), bt.size() * sizeof(int), cudaMemcpyHostToDevice));
  DIP_CUDA(cudaMemcpy(a->d_blk_start, bs.data(), bs.size() * sizeof(int), cudaMemcpyHostToDevice));
  DIP_CUDA(cudaMemcpy(a->d_numel, ne.data(), ne.size() * sizeof(int), cudaMemcpyHostToDevice));
  DIP_CUDA(cudaMemcpy(a->d_off, off.data(), off.size() * sizeof(long long), cudaMemcpyHostToDevice));
  *out = a;
  return 0;
}
void dip_adam_destroy(dip_adam* a) {
  if (!a) return;
  cudaFree(a->d_p); cudaFree(a->d_g); cudaFree(a->d_m); cudaFree(a->d_v);
  cudaFree(a->d_blk_tensor); cudaFree(a->d_blk_start); cudaFree(a->d_numel); cudaFree(a->d_off);
  delete a;
}
int dip_adam_bind(dip_adam* a, void* const* p, void* const* g, void* const* m, void* const* v) {
  DIP_CUDA(cudaMemcpy(a->d_p, p, a->n * sizeof(void*), cudaMemcpyHostToDevice));
  DIP_CUDA(cudaMemcpy(a->d_g, g, a->n * sizeof(void*), cudaMemcpyHostToDevice));
  DIP_CUDA(cudaMemcpy(a->d_m, m, a->n * sizeof(void*), cudaMemcpyHostToDevice));
  DIP_CUDA(cudaMemcpy(a->d_v, v, a->n * sizeof(void*), cudaMemcpyHostToDevice));
  a->bound = true;
  a->bind_gen++;
  return 0;
}
int dip_adam_step(dip_adam* a, double lr, double beta1, double beta2, double eps, int step, dip_stream_t stream) {
  if (!a->bound) return fail("dip_adam_step: not bound");
  if (step < 1) return fail("dip_adam_step: step must be >= 1");
  AdamTable t{a->d_p, a->d_g, a->d_m, a->d_v, a->d_blk_tensor, a->d_blk_start, a->d_numel, a->nblocks};
  launch_adam(t, lr, beta1, beta2, eps, step, nullptr, (cudaStream_t)stream);
  DIP_CUDA(cudaGetLastError());
  return 0;
}

// One iteration of the lean closure: noise -> forward -> MSE -> backward -> Adam.  With it_dev != nullptr every
// per-iteration scalar (Philox stream, loss slot, record slot, Adam step) comes from device counters, so the launch sequence
// is identical for every iteration and can be replayed as a CUDA graph.  track != nullptr adds the tracker's two kernels
// between the loss and the backward pass and steps Adam with its action; track->records is this call's first record.
static int run_body(dip_plan* P, dip_adam* adam, const float* z0, const float* target, const float* mask, float sigma,
                    uint64_t seed, int step_base, double lr, float* out, double* loss_slot, const dip_track* track, int* it_dev,
                    cudaStream_t s) {
  const size_t nz = (size_t)P->H * P->W * P->desc.in_channels;
  const int hw = P->H * P->W;
  const float* zin = z0;
  Recorder runner{&P->timer};   // the runner's own launches: timed like the plan's, not part of its forward / backward counts
  P->side_on = getenv("DIP_NO_SIDE") == nullptr;
  P->wev_used = 0;
  if (P->side_on && P->bound) {
    // weight repack on the side stream from the very start of the iteration (beside the noise kernel); plan_forward joins
    // it, and counts it as its own
    P->rec.n = 0;
    plan_pack(P, fork_side(P, s));
    P->prepacked = true;
  }
  if (sigma > 0.f && P->W % 4 != 0) {   // the fused k_noise_pad needs W % 4 == 0: separate k_noise + k_input_pad launches
    ENQ(&runner, hbm(H_NOISE, 0), 2.0 * nz * sizeof(float), s, launch_noise(z0, P->zbuf, sigma, seed, (uint64_t)step_base, it_dev, nz, s));
    zin = P->zbuf;
  } else if (sigma > 0.f) {
    P->fnoise.on = true; P->fnoise.z0 = z0; P->fnoise.sigma = sigma; P->fnoise.seed = seed; P->fnoise.offset = (uint64_t)step_base;
    P->fnoise.it_dev = it_dev;
  }
  const int frc = plan_forward(P, zin, nullptr, 0.f, out, s);
  P->fnoise.on = false;
  DIP_CHECK(frc);
  const int* slot_idx = it_dev != nullptr ? it_dev + 1 : nullptr;
  if (P->ds_K > 0) {
    // super-resolution: loss on the downsampled output (super-resolution.ipynb c10:8-11); the operator's adjoint
    // turns the low-resolution loss gradient into dL/d(out)
    const int co = P->desc.out_channels;
    ENQ(&runner, hbm(H_DOWN_FWD, 0), (double)co * ((double)P->H * P->W + (double)P->ds_Ho * P->ds_Wo) * sizeof(float), s,
        DIP_CUDA(launch_down_fwd(P->out_saved, co, P->H, P->W, P->ds_kern, P->ds_K, P->ds_f, P->ds_pad, P->ds_y, s)));
    launch_mse(P->ds_y, target, mask, co, P->ds_Ho * P->ds_Wo, loss_slot, P->ds_dy, slot_idx, s);
    ENQ(&runner, hbm(H_DOWN_BWD, 0), (double)co * ((double)P->H * P->W + (double)P->ds_Ho * P->ds_Wo) * sizeof(float), s,
        DIP_CUDA(launch_down_bwd(P->ds_dy, co, P->H, P->W, P->ds_kern, P->ds_K, P->ds_f, P->ds_pad, P->dout, s)));
  } else {
    ENQ(&runner, hbm(H_MSE, mask != nullptr), (3.0 * P->desc.out_channels + (mask != nullptr ? 1.0 : 0.0)) * hw * sizeof(float), s,
        launch_mse(P->out_saved, target, mask, P->desc.out_channels, hw, loss_slot, P->dout, slot_idx, s));
  }
  TrackState* tstate = track != nullptr ? (TrackState*)track->state : nullptr;
  if (track != nullptr) {
    const int n = P->desc.out_channels * hw;
    const bool gt = track->gt != nullptr;
    ENQ(&runner, hbm(H_TRACK_OUT, gt), (gt ? 4.0 : 3.0) * n * sizeof(float), s,
        launch_track_out(P->out_saved, (const float*)track->gt, (float*)track->out_avg, tstate, (float)track->exp_weight,
                         (float)(1.0 - track->exp_weight), n, track->records, slot_idx, s));
    ENQ(&runner, hbm(H_TRACK_DECIDE, 0), (kTrackRecord + 1.0) * sizeof(double) + 2.0 * sizeof(TrackState), s,
        launch_track_decide(loss_slot, track->records, tstate, track->show_every, track->backtrack_db, gt, slot_idx, s));
  }
  DIP_CHECK(plan_backward(P, P->dout, s));
  if (!adam->bound) return fail("dip_run_iterations: adam not bound");
  AdamTable t{adam->d_p, adam->d_g, adam->d_m, adam->d_v, adam->d_blk_tensor, adam->d_blk_start, adam->d_numel, adam->nblocks};
  {
    double np_ = 0; for (long long n : adam->numel) np_ += (double)n;
    if (track == nullptr)
      ENQ(&runner, hbm(H_ADAM, 0), 7.0 * np_ * sizeof(float), s, launch_adam(t, lr, 0.9, 0.999, 1e-8, step_base + 1, it_dev, s));
    else   // + the snapshot write of a save
      ENQ(&runner, hbm(H_ADAM_TRACK, 0), 8.0 * np_ * sizeof(float), s,
          launch_adam_track(t, lr, 0.9, 0.999, 1e-8, step_base + 1, it_dev, AdamTrack{tstate, (float*)track->snapshot, adam->d_off}, s));
  }
  if (it_dev != nullptr) launch_advance(it_dev, s);
  DIP_CUDA(cudaGetLastError());
  return 0;
}

size_t dip_track_state_bytes(void) { return sizeof(TrackState); }

static int check_track(const dip_track* t) {
  if (!(t->exp_weight >= 0.0 && t->exp_weight < 1.0))
    return fail("dip_run_iterations_tracked: exp_weight must be in [0, 1), got " + std::to_string(t->exp_weight));
  if (t->show_every < 0) return fail("dip_run_iterations_tracked: show_every must be >= 0, got " + std::to_string(t->show_every));
  if (t->backtrack_db != t->backtrack_db) return fail("dip_run_iterations_tracked: backtrack_db is NaN");
  if (t->out_avg == nullptr) return fail("dip_run_iterations_tracked: out_avg is NULL");
  if (t->snapshot == nullptr) return fail("dip_run_iterations_tracked: snapshot is NULL");
  if (t->state == nullptr) return fail("dip_run_iterations_tracked: state is NULL");
  if (t->records == nullptr) return fail("dip_run_iterations_tracked: records is NULL");
  return 0;
}

int dip_run_iterations_tracked(dip_plan* P, dip_adam* adam, const void* z0, const void* target, const void* mask, float sigma,
                               uint64_t seed, int step0, int iters, double lr, void* out, double* loss_hist,
                               const dip_track* track, dip_stream_t stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (track != nullptr) DIP_CHECK(check_track(track));
  if (iters <= 0) return 0;
  const bool use_graph = !P->timer.on && getenv("DIP_NO_GRAPH") == nullptr;
  if (!use_graph) {
    for (int i = 0; i < iters; ++i) {
      double* lp = loss_hist != nullptr ? loss_hist + i : P->loss_ring;
      DIP_CUDA(cudaMemsetAsync(lp, 0, sizeof(double), s));
      dip_track ti;
      if (track != nullptr) {
        ti = *track;
        ti.records = track->records + (size_t)kTrackRecord * i;
        DIP_CUDA(cudaMemsetAsync(ti.records, 0, kTrackRecord * sizeof(double), s));
      }
      DIP_CHECK(run_body(P, adam, (const float*)z0, (const float*)target, (const float*)mask, sigma, seed, step0 + i, lr,
                         (float*)out, lp, track != nullptr ? &ti : nullptr, nullptr, s));
    }
    return 0;
  }
  if (loss_hist == nullptr && iters > dip_plan::kLossRing) {
    // internal ring too small: split the call
    for (int done = 0; done < iters; done += dip_plan::kLossRing) {
      const int n = iters - done < dip_plan::kLossRing ? iters - done : dip_plan::kLossRing;
      dip_track tc;
      if (track != nullptr) { tc = *track; tc.records = track->records + (size_t)kTrackRecord * done; }
      DIP_CHECK(dip_run_iterations_tracked(P, adam, z0, target, mask, sigma, seed, step0 + done, n, lr, out, nullptr,
                                           track != nullptr ? &tc : nullptr, stream));
    }
    return 0;
  }
  // the legacy default stream cannot be captured: replay on a private stream, ordered against the caller's stream
  DIP_CHECK(ensure_gstream(P));
  cudaStream_t gs = P->gstream;
  DIP_CUDA(cudaEventRecord(P->gev_in, s));
  DIP_CUDA(cudaStreamWaitEvent(gs, P->gev_in, 0));
  double* slots = loss_hist != nullptr ? loss_hist : P->loss_ring;
  dip_plan::GraphKey key;
  key.z0 = z0; key.target = target; key.mask = mask; key.out = out; key.slots = slots;
  key.adam_id = adam->id; key.adam_bind = adam->bind_gen; key.sigma = sigma; key.seed = seed; key.lr = lr;
  if (track != nullptr) key.track = *track;
  if (P->gexec == nullptr || !(key == P->gkey)) {
    if (P->gexec != nullptr) { cudaGraphExecDestroy(P->gexec); P->gexec = nullptr; }
    DIP_CHECK(capture_graph(gs, &P->gexec, [&](cudaStream_t cs) {
      return run_body(P, adam, (const float*)z0, (const float*)target, (const float*)mask, sigma, seed, 0, lr, (float*)out, slots,
                      track, P->it_dev, cs);
    }));
    P->gkey = key;
  }
  const int init[2] = {step0, 0};
  DIP_CUDA(cudaMemcpyAsync(P->it_dev, init, sizeof init, cudaMemcpyHostToDevice, gs));
  DIP_CUDA(cudaMemsetAsync(slots, 0, (size_t)iters * sizeof(double), gs));
  if (track != nullptr) DIP_CUDA(cudaMemsetAsync(track->records, 0, (size_t)iters * kTrackRecord * sizeof(double), gs));
  for (int i = 0; i < iters; ++i) DIP_CUDA(cudaGraphLaunch(P->gexec, gs));
  DIP_CUDA(cudaEventRecord(P->gev_out, gs));
  DIP_CUDA(cudaStreamWaitEvent(s, P->gev_out, 0));
  return 0;
}

int dip_run_iterations(dip_plan* P, dip_adam* adam, const void* z0, const void* target, const void* mask, float sigma,
                       uint64_t seed, int step0, int iters, double lr, void* out, double* loss_hist, dip_stream_t stream) {
  return dip_run_iterations_tracked(P, adam, z0, target, mask, sigma, seed, step0, iters, lr, out, loss_hist, nullptr, stream);
}

int dip_input_grad(dip_plan* P, void* dz, dip_stream_t stream) {
  if (!P->desc.input_grad) return fail("dip_input_grad: the plan was created without input_grad");
  Level& v = P->lv[0];
  launch_input_grad(v.dPin, v.ns > 0 ? v.dS : nullptr, v.Cin, v.Cin_act, v.H, v.W, (float*)dz, (cudaStream_t)stream, P->zero_pad);
  DIP_CUDA(cudaGetLastError());
  return 0;
}

int dip_plan_buffer(const dip_plan* plan, const char* name, void** ptr, int* dims4) {
  auto it = plan->bufs.find(name);
  if (it == plan->bufs.end()) return fail(std::string("dip_plan_buffer: unknown buffer ") + name);
  *ptr = it->second.ptr;
  dims4[0] = it->second.rows; dims4[1] = it->second.cols; dims4[2] = it->second.ld; dims4[3] = it->second.c;
  return 0;
}
int dip_plan_set_timing(dip_plan* plan, int enable) {
  plan->timer.on = enable != 0;
  plan->timer.reset();
  return 0;
}
int dip_plan_get_timing(dip_plan* plan, double* ms3, double* flops3, int* launches3) {
  for (int i = 0; i < 3; ++i) { ms3[i] = 0; flops3[i] = 0; launches3[i] = 0; }
  for (const Timer::Rec& r : plan->timer.recs) {
    DIP_CUDA(cudaEventSynchronize(plan->timer.pool[r.e1]));
    float ms = 0.f;
    DIP_CUDA(cudaEventElapsedTime(&ms, plan->timer.pool[r.e0], plan->timer.pool[r.e1]));
    if (r.cls > 2) continue;   // HBM-bound kernels (class >= 16) are reported through dip_plan_get_timing_records only
    ms3[r.cls] += ms; flops3[r.cls] += r.flops; launches3[r.cls] += 1;
  }
  plan->timer.reset();
  return 0;
}
int dip_plan_get_timing_records(dip_plan* plan, int max_records, int* cls, double* flops, double* ms) {
  int n = 0;
  for (const Timer::Rec& r : plan->timer.recs) {
    if (n >= max_records) break;
    DIP_CUDA(cudaEventSynchronize(plan->timer.pool[r.e1]));
    float t = 0.f;
    DIP_CUDA(cudaEventElapsedTime(&t, plan->timer.pool[r.e0], plan->timer.pool[r.e1]));
    cls[n] = r.cls; flops[n] = r.flops; ms[n] = t;
    ++n;
  }
  plan->timer.reset();
  return n;
}
int dip_plan_num_launches(const dip_plan* plan, int* fwd, int* bwd) {
  *fwd = plan->launches_fwd; *bwd = plan->launches_bwd;
  return 0;
}

// ---------------------------------------------------------------------------------------------- single-op entry points
size_t dip_op_scratch_bytes(void) { return (size_t)96 << 20; }

// Sets up one convolution that an entry point has described (shapes, tensors and which of do_fprop / has_dgrad /
// do_wgrad it runs) in the caller's scratch area, laid out as [fprop pack | dgrad pack | PackEntry | UnpackEntry | wgrad
// partials | bf16 copies of dY and of the input (precision bf16)].  Operands whose layout does not fit are refused before
// anything is launched.  Then packs w, uploads the table entries, writes the bf16 copies and encodes the tensor maps.
static int op_setup(const char* name, ConvOp& op, int prec, const float* w, float* dw, void* scratch, cudaStream_t s) {
  DIP_CHECK(engine_init());
  const int max_c = op.do_fprop ? 256 : 160;   // dgrad / wgrad: the register accumulators hold at most 160 columns
  if (op.N != 128) return fail(std::string(name) + ": N must be 128");
  if (op.C % 4 != 0 || op.C > max_c)
    return fail(std::string(name) + ": C must be a multiple of 4 and <= " + std::to_string(max_c));
  op.bf16 = prec == DIP_PRECISION_BF16;
  op.set_shapes();
  const bool pack = op.do_fprop || op.has_dgrad;
  const bool cast_dy = op.bf16 && (op.has_dgrad || op.do_wgrad), cast_in = op.bf16 && (op.do_fprop || op.do_wgrad);
  if (cast_in) op.in_ld16 = round_up(op.in_ld, 8);
  Arena A{(uint8_t*)scratch};
  op.wp_f = op.do_fprop ? A.get<float>(op.wp_f_elems()) : nullptr;
  op.wp_d = op.has_dgrad ? A.get<float>(op.wp_d_elems()) : nullptr;
  PackEntry* d_pack = pack ? A.get<PackEntry>(1) : nullptr;
  UnpackEntry* d_unpack = op.do_wgrad ? A.get<UnpackEntry>(1) : nullptr;
  op.partial = op.do_wgrad ? A.get<float>(op.partial_elems(prec)) : nullptr;
  const long long dy_px = (long long)op.out_h * op.out_w, in_px = (long long)op.in_rows * op.in_cols;
  uint16_t* dy16 = cast_dy ? A.get<uint16_t>(dy_px * op.N) : nullptr;
  uint16_t* in16 = cast_in ? A.get<uint16_t>(in_px * op.in_ld16) : nullptr;
  if (A.off > dip_op_scratch_bytes())
    return fail(std::string(name) + ": the operands need " + std::to_string((A.off + (1 << 20) - 1) >> 20) +
                " MB of scratch, more than dip_op_scratch_bytes() = " + std::to_string(dip_op_scratch_bytes() >> 20) + " MB");
  if (pack) {
    const PackEntry e = op.pack_entry(prec, w);
    DIP_CUDA(cudaMemcpyAsync(d_pack, &e, sizeof e, cudaMemcpyHostToDevice, s));
    launch_k(k_pack_table, dim3(64, 1), dim3(256), 0, s, 1, (const PackEntry*)d_pack);
  }
  if (op.do_wgrad) {
    const UnpackEntry e = op.unpack_entry(prec, dw);
    DIP_CUDA(cudaMemcpyAsync(d_unpack, &e, sizeof e, cudaMemcpyHostToDevice, s));
    op.unpack = d_unpack;
  }
  if (cast_dy) launch_cast_bf16(op.dy, op.N, op.N, dy_px, Twin{dy16, op.N}, s);
  if (cast_in) launch_cast_bf16(op.in, op.in_ld, op.in_ld, in_px, Twin{in16, op.in_ld16}, s);
  op.dy16 = dy16; op.in16 = in16;
  DIP_CUDA(cudaGetLastError());
  return is_tc(prec) ? op.build_tc() : 0;
}

int dip_op_conv_fprop(const void* a, int a_h, int a_w, int a_c, const void* w, const void* bias, int N, int C, int k, int stride,
                      int offx, int offy, int rot, void* d, int d_h, int d_w, double* stats, int precision, void* scratch,
                      dip_stream_t stream) {
  cudaStream_t s = (cudaStream_t)stream;
  ConvOp op;
  op.N = N; op.C = C; op.k = k; op.stride = stride; op.rot = rot;
  op.do_fprop = true; op.has_dgrad = false; op.do_wgrad = false;
  op.in = (const float*)a; op.in_rows = a_h; op.in_cols = a_w; op.in_ld = a_c; op.offx = offx; op.offy = offy;
  op.out = (float*)d; op.out_h = d_h; op.out_w = d_w; op.stats = stats;
  DIP_CHECK(op_setup("dip_op_conv_fprop", op, precision, (const float*)w, nullptr, scratch, s));
  return op.run_fprop(precision, (const float*)bias, s);
}
int dip_op_conv_dgrad(const void* dy, int dy_h, int dy_w, const void* w, int N, int C, int k, int rot, void* dx, int dx_h, int dx_w,
                      int precision, void* scratch, dip_stream_t stream) {
  cudaStream_t s = (cudaStream_t)stream;
  ConvOp op;
  op.N = N; op.C = C; op.k = k; op.rot = rot;
  op.do_fprop = false; op.has_dgrad = true; op.do_wgrad = false;
  op.dy = (const float*)dy; op.out_h = dy_h; op.out_w = dy_w;
  op.dg_out = (float*)dx; op.dg_out_h = dx_h; op.dg_out_w = dx_w; op.dg_off = -(k - 1);
  DIP_CHECK(op_setup("dip_op_conv_dgrad", op, precision, (const float*)w, nullptr, scratch, s));
  return op.run_dgrad(precision, s);
}
int dip_op_conv_dgrad_s2(const void* dy, int dy_h, int dy_w, const void* w, int N, int C, int rot, void* dx, int precision,
                         void* scratch, dip_stream_t stream) {
  cudaStream_t s = (cudaStream_t)stream;
  ConvOp op;
  op.N = N; op.C = C; op.k = 3; op.stride = 2; op.rot = rot;
  op.do_fprop = false; op.has_dgrad = true; op.do_wgrad = false;
  op.dg_s2 = true;
  op.dy = (const float*)dy; op.out_h = dy_h; op.out_w = dy_w;
  op.dg_out = (float*)dx; op.dg_out_h = 2 * dy_h + 2; op.dg_out_w = 2 * dy_w + 2; op.dg_off = -2;
  DIP_CHECK(op_setup("dip_op_conv_dgrad_s2", op, precision, (const float*)w, nullptr, scratch, s));
  return op.run_dgrad(precision, s);
}
int dip_op_conv_wgrad(const void* dy, int dy_h, int dy_w, const void* a, int a_h, int a_w, int a_c, int N, int C, int k, int stride,
                      int offx, int offy, int rot, void* dw, int precision, void* scratch, dip_stream_t stream) {
  cudaStream_t s = (cudaStream_t)stream;
  ConvOp op;
  op.N = N; op.C = C; op.k = k; op.stride = stride; op.rot = rot;
  op.do_fprop = false; op.has_dgrad = false; op.do_wgrad = true;
  op.in = (const float*)a; op.in_rows = a_h; op.in_cols = a_w; op.in_ld = a_c; op.offx = offx; op.offy = offy;
  op.dy = (const float*)dy; op.out_h = dy_h; op.out_w = dy_w;
  DIP_CHECK(op_setup("dip_op_conv_wgrad", op, precision, nullptr, (float*)dw, scratch, s));
  return op.run_wgrad(precision, s);
}

}  // extern "C"
