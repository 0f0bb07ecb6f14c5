// HBM-bound kernels of the dip-b200 engine: coalesced, 128-bit vectorised NHWC fp32.
//
// Each kernel replaces a chain of torch ops of the reference's skip network
// (models/skip.py:41-100 built from models/common.py:76-124):
//   input_pad        : net_input perturbation + nn.ReflectionPad2d(1)            (denoising.ipynb c10:12-13, common.py:117)
//   bn_act_write     : nn.BatchNorm2d (training mode) + nn.LeakyReLU(0.2) + nn.ReflectionPad2d(1)   (common.py:96,82,117)
//                      (pad != 'reflection': the zero halo of Conv2d(padding=1) instead, in every halo writer / fold below;
//                       act_fun 'Swish' / 'ELU' / 'none' (common.py:76-92) instead of LeakyReLU in every BN(+act) kernel)
//   bn_act_head      : last BN + LeakyReLU + 1x1 conv 128->3 + nn.Sigmoid in one pass (skip.py:90-98)
//   cat_stats/write  : nn.Upsample(x2) + Concat + nn.BatchNorm2d(132) + pad     (skip.py:81,50-55; common.py:19-39)
//   bn_bwd_*/cat_bwd_*: autograd adjoints of the above, with the producer of the incoming gradient fused in
//                       (reflection-pad adjoint, upsample adjoint, skip-conv dgrad, RGB-head dgrad+wgrad)
//   skinny_*         : 1x1 convs with <= 4 outputs (skip branches, skip.py:57-60)
//   mse / adam / noise: torch.nn.MSELoss, torch.optim.Adam.step, noise.normal_()  (common_utils.py:225-230)
#include "kernels.cuh"

#include <cuda_bf16.h>
#include <math_constants.h>
#include <math.h>
#include <stdlib.h>

#include <map>
#include <type_traits>
#include <utility>


namespace dip {

// items in flight per thread (item_loop) of the kernels whose gradient source is a reflection-pad fold: tuning knobs
#ifndef DIP_U_BWD1
#define DIP_U_BWD1 4
#endif
#ifndef DIP_U_CATBWD
#define DIP_U_CATBWD 2
#endif
#ifndef DIP_U_HEAD
#define DIP_U_HEAD 4       // pixels in flight per warp of the fused BN + RGB head kernel
#endif
#ifndef DIP_CAT_MINBLOCKS
#define DIP_CAT_MINBLOCKS 4   // __launch_bounds__ min blocks per SM of the concat kernels (register cap 64: level-0 k_cat_write 62 -> 49.5 us; 5 spills)
#endif

// ------------------------------------------------------------------------------------------------ helpers
__device__ __forceinline__ int reflect_idx(int i, int n) {
  if (i < 0) i = -i;
  if (i >= n) i = 2 * n - 2 - i;
  return i;
}
__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ float4 f4add(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
__device__ __forceinline__ float4 f4fma(float w, float4 a, float4 acc) {
  return make_float4(fmaf(w, a.x, acc.x), fmaf(w, a.y, acc.y), fmaf(w, a.z, acc.z), fmaf(w, a.w, acc.w));
}
__device__ __forceinline__ float4 f4mul(float4 a, float4 b) { return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w); }
__device__ __forceinline__ float4 f4mla(float4 a, float4 b, float4 acc) {
  return make_float4(fmaf(a.x, b.x, acc.x), fmaf(a.y, b.y, acc.y), fmaf(a.z, b.z, acc.z), fmaf(a.w, b.w, acc.w));
}
// 4 consecutive channels as bf16 (round to nearest even), one 8-byte store
__device__ __forceinline__ void st4_bf16(uint16_t* p, float4 v) {
  const __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
  uint2 u;
  u.x = *reinterpret_cast<const uint32_t*>(&a);
  u.y = *reinterpret_cast<const uint32_t*>(&b);
  *reinterpret_cast<uint2*>(p) = u;
}
__device__ __forceinline__ uint16_t bf16_bits(float x) {
  const __nv_bfloat16 h = __float2bfloat16_rn(x);
  return *reinterpret_cast<const uint16_t*>(&h);
}
__device__ __forceinline__ float4 f4zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ float f4dot(float4 a, float4 b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }
// The activation f of every BN(+act) stage and its adjoint g * f'(y), both of the fp32 pre-activation y = fma(x, scale, shift)
// (ACT: kAct*).  Swish's sigmoid is 1 / (1 + e^-y), which tends to 0 or 1 for large |y| without an inf / inf or 0 * inf.
template <int ACT>
__device__ __forceinline__ float act_fwd(float y) {
  if constexpr (ACT == kActSwish) return y * (1.f / (1.f + expf(-y)));
  else if constexpr (ACT == kActElu) return y > 0.f ? y : expm1f(y);
  else if constexpr (ACT == kActNone) return y;
  else return y > 0.f ? y : kLreluSlope * y;
}
template <int ACT>
__device__ __forceinline__ float act_bwd(float y, float g) {
  if constexpr (ACT == kActSwish) {
    const float s = 1.f / (1.f + expf(-y));
    return g * (s * (1.f + y * (1.f - s)));
  } else if constexpr (ACT == kActElu) {
    return y > 0.f ? g : g * expf(y);
  } else if constexpr (ACT == kActNone) {
    return g;
  } else {
    return y > 0.f ? g : kLreluSlope * g;
  }
}
template <int ACT>
__device__ __forceinline__ float4 act_fwd4(float4 y) {
  return make_float4(act_fwd<ACT>(y.x), act_fwd<ACT>(y.y), act_fwd<ACT>(y.z), act_fwd<ACT>(y.w));
}
template <int ACT>
__device__ __forceinline__ float4 act_bwd4(float4 y, float4 g) {
  return make_float4(act_bwd<ACT>(y.x, g.x), act_bwd<ACT>(y.y, g.y), act_bwd<ACT>(y.z, g.z), act_bwd<ACT>(y.w, g.w));
}
// the kernel instantiation for a plan's activation kind: pick(std::integral_constant<int, ACT>) returns it
template <class Pick>
static auto act_pick(int act_fun, Pick pick) {
  switch (act_fun) {
    case kActSwish: return pick(std::integral_constant<int, kActSwish>());
    case kActElu: return pick(std::integral_constant<int, kActElu>());
    case kActNone: return pick(std::integral_constant<int, kActNone>());
    default: return pick(std::integral_constant<int, kActLeakyRelu>());
  }
}
__device__ __forceinline__ float4 shfl_xor4(float4 a, int o) {
  return make_float4(__shfl_xor_sync(0xffffffffu, a.x, o), __shfl_xor_sync(0xffffffffu, a.y, o),
                     __shfl_xor_sync(0xffffffffu, a.z, o), __shfl_xor_sync(0xffffffffu, a.w, o));
}

static constexpr int kMaxBnC = 264;   // widest BatchNorm: the 256-channel concat of the skip=128 configuration
// per-thread BN coefficients for channels 4v..4v+3
struct Bn4 {
  float4 mean, rstd, scale, shift;
};
// Block-cooperative: thread c (< C) evaluates channel c once in fp64 (sum of the accumulator replicas -> mean, rstd),
// the coefficients are broadcast through shared memory as float4s.  Every thread of the block must call it (barrier);
// TAG distinguishes the static buffers when a kernel needs two BatchNorms.  v < 0: this thread needs no coefficients.
template <int TAG>
__device__ __forceinline__ Bn4 bn_coef(const BnRef& bn, int v) {
  __shared__ __align__(16) float s_mean[kMaxBnC], s_rstd[kMaxBnC], s_scale[kMaxBnC], s_shift[kMaxBnC];
  for (int c = threadIdx.x; c < bn.C; c += blockDim.x) {
    const int ct = (c + bn.rot) % bn.C;
    const double m = acc_get(bn.fwd + c * kAccS) * static_cast<double>(bn.inv_n);
    double var = acc_get(bn.fwd + (bn.C + c) * kAccS) * static_cast<double>(bn.inv_n) - m * m;
    if (var < 0.0) var = 0.0;
    const float mean = static_cast<float>(m);
    const float rstd = static_cast<float>(1.0 / sqrt(var + static_cast<double>(kBnEps)));
    const float sc = bn.gamma[ct] * rstd;
    s_mean[c] = mean;
    s_rstd[c] = rstd;
    s_scale[c] = sc;
    s_shift[c] = bn.beta[ct] - mean * sc;
  }
  __syncthreads();
  Bn4 r;
  if (v >= 0 && 4 * v + 3 < bn.C) {
    r.mean = *reinterpret_cast<const float4*>(&s_mean[4 * v]);
    r.rstd = *reinterpret_cast<const float4*>(&s_rstd[4 * v]);
    r.scale = *reinterpret_cast<const float4*>(&s_scale[4 * v]);
    r.shift = *reinterpret_cast<const float4*>(&s_shift[4 * v]);
  } else {
    r.mean = r.rstd = r.scale = r.shift = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  return r;
}
// means of the backward sums (sum dz / n, sum dz*xhat / n), block-cooperative like bn_coef
template <int TAG>
__device__ __forceinline__ void bwd_means(const double* __restrict__ bwd, int C, float inv_n, int v, float4& m1, float4& m2) {
  __shared__ __align__(16) float s_m1[kMaxBnC], s_m2[kMaxBnC];
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    s_m1[c] = static_cast<float>(acc_get(bwd + c * kAccS) * inv_n);
    s_m2[c] = static_cast<float>(acc_get(bwd + (C + c) * kAccS) * inv_n);
  }
  __syncthreads();
  m1 = *reinterpret_cast<const float4*>(&s_m1[4 * v]);
  m2 = *reinterpret_cast<const float4*>(&s_m2[4 * v]);
}
__device__ __forceinline__ float4 bn_apply(const Bn4& c, float4 x) {
  return make_float4(fmaf(x.x, c.scale.x, c.shift.x), fmaf(x.y, c.scale.y, c.shift.y), fmaf(x.z, c.scale.z, c.shift.z),
                     fmaf(x.w, c.scale.w, c.shift.w));
}
__device__ __forceinline__ float4 bn_xhat(const Bn4& c, float4 x) {
  return make_float4((x.x - c.mean.x) * c.rstd.x, (x.y - c.mean.y) * c.rstd.y, (x.z - c.mean.z) * c.rstd.z,
                     (x.w - c.mean.w) * c.rstd.w);
}

// Launch geometry for "vec-lane per 4 channels" kernels: thread = (item slot, v); v fixed per thread.
struct VecGeom {
  int VL, PPB, threads, blocks;
};
static VecGeom vec_geom(int C, long long nitems) {
  VecGeom g;
  g.VL = C / 4;
  g.PPB = 256 / g.VL;
  if (g.PPB < 1) g.PPB = 1;
  g.threads = g.VL * g.PPB;
  long long nb = (nitems + g.PPB - 1) / g.PPB;
  const long long cap = g.VL >= 8 ? kNumSms * 8 : kNumSms * 2;
  g.blocks = static_cast<int>(nb < cap ? nb : cap);
  if (g.blocks < 1) g.blocks = 1;
  return g;
}

// Block reduction of K float4 accumulators over the item slots of the block, then fp64 atomics into dst[k][c].
// Threads are laid out tid = slot * VL + v.  For VL in {1,2,4,8,16} the lanes that share v are first folded with
// warp shuffles (blockDim is then a multiple of 32).  wid[k] = valid channels of dst[k].
// The accumulators live one per 128-byte line (kAccS): hundreds of blocks add to the same 2*C addresses at the end of a
// single-wave kernel, and neighbouring channels sharing an L2 atomic unit serialise their atomics.
template <int K>
__device__ __forceinline__ void block_reduce_atomic(float4 (&acc)[K], int VL, int PPB, double* const* dst, const int* wid) {
  extern __shared__ float4 red_smem[];
  const int tid = threadIdx.x;
  int nparts, part;
  if (VL < 32 && (VL & (VL - 1)) == 0) {
    for (int o = 16; o >= VL; o >>= 1) {
#pragma unroll
      for (int k = 0; k < K; ++k) acc[k] = f4add(acc[k], shfl_xor4(acc[k], o));
    }
    nparts = blockDim.x >> 5;
    part = tid >> 5;
    if ((tid & 31) < VL) {
#pragma unroll
      for (int k = 0; k < K; ++k) red_smem[(k * nparts + part) * VL + (tid & 31)] = acc[k];
    }
  } else {
    nparts = PPB;
    part = tid / VL;
    if (part < nparts) {
#pragma unroll
      for (int k = 0; k < K; ++k) red_smem[(k * nparts + part) * VL + (tid % VL)] = acc[k];
    }
  }
  __syncthreads();
  // one (k, v) pair per thread (K <= PPB always): the column is summed in fp64 and added to the global accumulators
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const int v = tid - k * VL;
    if (v < 0 || v >= VL || dst[k] == nullptr) continue;
    double sv[4] = {0.0, 0.0, 0.0, 0.0};
    for (int pp = 0; pp < nparts; ++pp) {
      const float4 t = red_smem[(k * nparts + pp) * VL + v];
      sv[0] += t.x; sv[1] += t.y; sv[2] += t.z; sv[3] += t.w;
    }
#pragma unroll
    for (int e = 0; e < 4; ++e)
      if (4 * v + e < wid[k]) atomicAdd(dst[k] + (4 * v + e) * kAccS + (blockIdx.x % kAccR) * kAccLine, sv[e]);
  }
}
static size_t red_bytes(const VecGeom& g, int K) {
  return static_cast<size_t>(K) * g.threads * sizeof(float4);
}
template <class... KArgs, class... Args>
static void launch_red(void (*kernel)(KArgs...), int blocks, int threads, size_t smem, cudaStream_t s, Args... args) {
  launch_k(kernel, dim3(blocks), dim3(threads), smem, s, 1, args...);
}
// Grid-stride kernels get exactly one resident wave (no tail wave): blocks = min(needed, SMs * occupancy).
template <class Kern>
static void fit_grid(VecGeom& g, Kern kernel, size_t smem) {
  static std::map<std::pair<const void*, int>, int> cache;
  const std::pair<const void*, int> key(reinterpret_cast<const void*>(kernel), g.threads);
  auto it = cache.find(key);
  int per_sm;
  if (it == cache.end()) {
    per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, g.threads, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
    cache[key] = per_sm;
  } else {
    per_sm = it->second;
  }
  const int cap = kNumSms * per_sm;
  if (g.blocks > cap) g.blocks = cap;
}

// ------------------------------------------------------------------------------------------------ input_pad
// ZP (zero padding, Conv2d(padding=1)): the halo ring is written as zeros instead of the mirrored pixels.  Every kernel
// that writes or folds a halo takes ZP as a template parameter, so the reflection instantiation is the unchanged code.
template <bool ZP>
__global__ void k_input_pad(const float* __restrict__ z, const float* __restrict__ noise, float sigma,
                            float* __restrict__ dst, int C, int H, int W, int Cs, Twin t16) {
  pdl_enter();
  __shared__ float tile[32][33];
  const int Wp = W + 2;
  const int yy = blockIdx.y;
  const int sy = ZP ? yy - 1 : reflect_idx(yy - 1, H);
  const int tx = threadIdx.x, ty = threadIdx.y;
  for (int c0 = 0; c0 < C; c0 += 32) {
    const int xx = blockIdx.x * 32 + tx;
    for (int k = 0; k < 4; ++k) {
      const int c = c0 + ty + 8 * k;
      float val = 0.f;
      if (xx < Wp && c < Cs && (!ZP || (sy >= 0 && sy < H && xx >= 1 && xx <= W))) {
        const int sx = ZP ? xx - 1 : reflect_idx(xx - 1, W);
        const size_t off = (static_cast<size_t>(c) * H + sy) * W + sx;
        val = z[off];
        if (noise != nullptr) val = fmaf(noise[off], sigma, val);
      }
      tile[ty + 8 * k][tx] = val;
    }
    __syncthreads();
    for (int k = 0; k < 4; ++k) {
      const int xo = blockIdx.x * 32 + ty + 8 * k;
      const int c = c0 + tx;
      if (xo < Wp && c < C) {
        dst[(static_cast<size_t>(yy) * Wp + xo) * C + c] = tile[tx][ty + 8 * k];
        if (t16.p != nullptr) t16.p[(static_cast<size_t>(yy) * Wp + xo) * t16.ld + c] = bf16_bits(tile[tx][ty + 8 * k]);
      }
    }
    __syncthreads();
  }
}
void launch_input_pad(const float* z, const float* noise, float sigma, float* dst, int C, int H, int W,
                      cudaStream_t s, int c_src, Twin t16, int zero_pad) {
  dim3 grid((W + 2 + 31) / 32, H + 2), block(32, 8);
  launch_k(zero_pad ? k_input_pad<true> : k_input_pad<false>, dim3(grid), dim3(block), 0, s, 1, z, noise, sigma, dst, C, H, W,
           c_src > 0 ? c_src : C, t16);
}

// ------------------------------------------------------------------------------------------------ cast (single ops)
__global__ void __launch_bounds__(256) k_cast_bf16(const float* __restrict__ x, int ld, int c4, long long n4, Twin t) {
  pdl_enter();
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long p = i / c4;
    const int v = static_cast<int>(i - p * c4);
    st4_bf16(t.p + p * t.ld + 4 * v, ld4(x + p * ld + 4 * v));
  }
}
void launch_cast_bf16(const float* x, int ld, int c, long long npix, Twin t, cudaStream_t s) {
  const long long n4 = npix * (c / 4);
  long long blocks = (n4 + 255) / 256;
  if (blocks > kNumSms * 8) blocks = kNumSms * 8;
  if (blocks < 1) blocks = 1;
  launch_k(k_cast_bf16, dim3((unsigned)blocks), dim3(256), 0, s, 1, x, ld, c / 4, n4, t);
}

// ------------------------------------------------------------------------------------------------ item loop
// Grid-stride loop with U independent items in flight per thread: all loads of the U items are issued before any of
// them is consumed (memory-level parallelism is what these latency-bound streaming kernels lack otherwise).
template <int U, class Load, class Use>
__device__ __forceinline__ void item_loop(int first, int stride, int n, Load load, Use use) {
  for (int p0 = first; p0 < n; p0 += U * stride) {
    decltype(load(0)) d[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int p = p0 + u * stride;
      if (p < n) d[u] = load(p);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int p = p0 + u * stride;
      if (p < n) use(p, d[u]);
    }
  }
}

// ------------------------------------------------------------------------------------------------ channel_stats
__global__ void __launch_bounds__(256) k_channel_stats(const float* __restrict__ x, int ld, int VL, int PPB, int npix,
                                                       double* __restrict__ fwd, int C) {
  pdl_enter();
  const int v = threadIdx.x % VL, slot = threadIdx.x / VL;
  float4 acc[2] = {f4zero(), f4zero()};
  item_loop<4>(blockIdx.x * PPB + slot, gridDim.x * PPB, npix,
               [&](int p) { return ld4(x + static_cast<size_t>(p) * ld + 4 * v); },
               [&](int, float4 t) {
                 acc[0] = f4add(acc[0], t);
                 acc[1] = f4mla(t, t, acc[1]);
               });
  double* const dst[2] = {fwd, fwd + C * kAccS};
  const int wid[2] = {C, C};
  block_reduce_atomic<2>(acc, VL, PPB, dst, wid);
}
void launch_channel_stats(const float* x, int ld, int C, int npix, double* fwd, cudaStream_t s) {
  VecGeom g = vec_geom(C, npix);
  fit_grid(g, k_channel_stats, red_bytes(g, 2));
  launch_red(k_channel_stats, g.blocks, g.threads, red_bytes(g, 2), s, x, ld, g.VL, g.PPB, npix, fwd, C);
}

// ------------------------------------------------------------------------------------------------ bn_act_write
// ZP: with pad, the halo cells are written as 0 (their load reads the nearest interior pixel, whose value is discarded)
// ACT: the activation applied when act != 0 (kAct*; like ZP a template parameter, so the LeakyReLU instantiations of
// this kernel and of the other BN(+act) kernels below are the unchanged code)
template <bool ZP, int ACT>
__global__ void __launch_bounds__(256) k_bn_act_write(const float* __restrict__ raw, int ld_in, BnRef bn, int H, int W,
                                                      float* __restrict__ dst, int ld_out, int pad, int act, int VL,
                                                      int PPB, Twin t16) {
  pdl_enter();
  const int v = threadIdx.x % VL, slot = threadIdx.x / VL;
  const Bn4 cf = bn_coef<0>(bn, v);
  const int Ho = H + 2 * pad, Wo = W + 2 * pad;
  item_loop<4>(blockIdx.x * PPB + slot, gridDim.x * PPB, Ho * Wo,
               [&](int p) {
                 const int yo = p / Wo, xo = p - yo * Wo;
                 const int yi = pad ? (ZP ? min(max(yo - 1, 0), H - 1) : reflect_idx(yo - 1, H)) : yo;
                 const int xi = pad ? (ZP ? min(max(xo - 1, 0), W - 1) : reflect_idx(xo - 1, W)) : xo;
                 return ld4(raw + (static_cast<size_t>(yi) * W + xi) * ld_in + 4 * v);
               },
               [&](int p, float4 x) {
                 float4 y = bn_apply(cf, x);
                 if (act) y = act_fwd4<ACT>(y);
                 if (ZP && pad) {
                   const int yo = p / Wo, xo = p - yo * Wo;
                   if (yo == 0 || yo == Ho - 1 || xo == 0 || xo == Wo - 1) y = f4zero();
                 }
                 if (dst != nullptr) st4(dst + static_cast<size_t>(p) * ld_out + 4 * v, y);
                 if (t16.p != nullptr) st4_bf16(t16.p + static_cast<size_t>(p) * t16.ld + 4 * v, y);
               });
}
void launch_bn_act_write(const float* raw, int ld_in, BnRef bn, int H, int W, float* dst, int ld_out, int pad,
                         int act, int act_fun, cudaStream_t s, Twin t16, int zero_pad) {
  VecGeom g = vec_geom(bn.C, static_cast<long long>(H + 2 * pad) * (W + 2 * pad));
  auto kernel = act_pick(act_fun, [&](auto a) {
    constexpr int A = decltype(a)::value;
    return zero_pad && pad ? k_bn_act_write<true, A> : k_bn_act_write<false, A>;
  });
  fit_grid(g, kernel, 0);
  launch_k(kernel, dim3(g.blocks), dim3(g.threads), 0, s, 1, raw, ld_in, bn, H, W, dst, ld_out, pad, act, g.VL, g.PPB, t16);
}

// BN + activation + RGB head + sigmoid: one warp per pixel (C = 128 -> 32 lanes x float4), nothing but out is written.
template <int ACT>
__global__ void __launch_bounds__(256) k_bn_act_head(const float* __restrict__ raw, BnRef bn, int npix, HeadRef head) {
  pdl_enter();
  const int lane = threadIdx.x & 31, wslot = threadIdx.x >> 5;
  const Bn4 cf = bn_coef<0>(bn, lane);
  float4 w[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) w[k] = k < head.K ? ld4(head.w + k * 128 + 4 * lane) : f4zero();
  const float hbk = ((lane >> 3) & 3) < head.K ? head.b[(lane >> 3) & 3] : 0.f;   // bias of the output this lane ends up with
  item_loop<DIP_U_HEAD>(blockIdx.x * 8 + wslot, gridDim.x * 8, npix,
               [&](int p) { return ld4(raw + static_cast<size_t>(p) * 128 + 4 * lane); },
               [&](int p, float4 x) {
                 const float4 y = act_fwd4<ACT>(bn_apply(cf, x));
                 float d[4];
#pragma unroll
                 for (int k = 0; k < 4; ++k) d[k] = f4dot(y, w[k]);
                 // 4 values x 32 lanes -> 4 totals in 6 shuffles (value-halving butterfly): after the xor-16 / xor-8 steps a
                 // lane carries output k = 2 * bit4 + bit3 of its lane index; the last three steps fold the 8 lanes of a group
                 const bool hi16 = (lane & 16) != 0, hi8 = (lane & 8) != 0;
                 float a0 = hi16 ? d[2] : d[0], a1 = hi16 ? d[3] : d[1];
                 a0 += __shfl_xor_sync(0xffffffffu, hi16 ? d[0] : d[2], 16);
                 a1 += __shfl_xor_sync(0xffffffffu, hi16 ? d[1] : d[3], 16);
                 float t = hi8 ? a1 : a0;
                 t += __shfl_xor_sync(0xffffffffu, hi8 ? a0 : a1, 8);
                 t += __shfl_xor_sync(0xffffffffu, t, 4);
                 t += __shfl_xor_sync(0xffffffffu, t, 2);
                 t += __shfl_xor_sync(0xffffffffu, t, 1);
                 const int k = (lane >> 3) & 3;
                 if ((lane & 7) == 0 && k < head.K) {
                   t += hbk;
                   head.out[static_cast<size_t>(k) * npix + p] = head.sigmoid ? 1.f / (1.f + expf(-t)) : t;
                 }
               });
}
void launch_bn_act_head(const float* raw, BnRef bn, int H, int W, HeadRef head, int act_fun, cudaStream_t s) {
  const int npix = H * W;
  int blocks = (npix + 7) / 8;
  if (blocks > kNumSms * 8) blocks = kNumSms * 8;
  auto kernel = act_pick(act_fun, [](auto a) { return k_bn_act_head<decltype(a)::value>; });
  launch_k(kernel, dim3(blocks), dim3(256), 0, s, 1, raw, bn, npix, head);
}

// ------------------------------------------------------------------------------------------------ concat stage
// Work item = one SOURCE pixel (si, sj) of U (h x w) and its 2x2 block of output pixels (2si+a, 2sj+b):
// 9 loads produce 4 upsampled values (bilinear, align_corners=False: weights 1/4, 3/4, edge clamp).
struct CatLane {
  int is_up;
  Bn4 bs;  // skip-branch BN (valid when !is_up)
};
__device__ __forceinline__ CatLane cat_lane(const CatArgs& a, int v) {
  CatLane l;
  l.is_up = v < a.Cu / 4;
  l.bs = bn_coef<1>(a.bn_s, l.is_up ? -1 : v - a.Cu / 4);
  return l;
}
// out[0..3] = pre-BN concat values at (2si,2sj), (2si,2sj+1), (2si+1,2sj), (2si+1,2sj+1) (skip branch: activation ACT)
template <int ACT>
__device__ __forceinline__ void cat_quad(const CatArgs& a, const CatLane& l, int si, int sj, int v, float4 (&out)[4]) {
  const int h = a.H >> 1, w = a.W >> 1;
  if (l.is_up) {
    const float* base = a.U + 4 * v;
    if (!a.bilinear) {
      const float4 c = ld4(base + (static_cast<size_t>(si) * w + sj) * a.Cu);
      out[0] = out[1] = out[2] = out[3] = c;
      return;
    }
    const int r0 = max(si - 1, 0), r2 = min(si + 1, h - 1);
    const int c0 = max(sj - 1, 0), c2 = min(sj + 1, w - 1);
    const int rr[3] = {r0, si, r2};
    float4 hl[3], hr[3];
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      const float* rowp = base + static_cast<size_t>(rr[q]) * w * a.Cu;
      const float4 n0 = ld4(rowp + static_cast<size_t>(c0) * a.Cu);
      const float4 n1 = ld4(rowp + static_cast<size_t>(sj) * a.Cu);
      const float4 n2 = ld4(rowp + static_cast<size_t>(c2) * a.Cu);
      hl[q] = f4fma(0.25f, n0, f4fma(0.75f, n1, f4zero()));
      hr[q] = f4fma(0.25f, n2, f4fma(0.75f, n1, f4zero()));
    }
    out[0] = f4fma(0.25f, hl[0], f4fma(0.75f, hl[1], f4zero()));
    out[1] = f4fma(0.25f, hr[0], f4fma(0.75f, hr[1], f4zero()));
    out[2] = f4fma(0.25f, hl[2], f4fma(0.75f, hl[1], f4zero()));
    out[3] = f4fma(0.25f, hr[2], f4fma(0.75f, hr[1], f4zero()));
  } else {
    const float* base = a.raw_s + 4 * (v - a.Cu / 4);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int i = 2 * si + (q >> 1), j = 2 * sj + (q & 1);
      out[q] = act_fwd4<ACT>(bn_apply(l.bs, ld4(base + (static_cast<size_t>(i) * a.W + j) * a.Cs)));
    }
  }
}

template <int ACT>
__global__ void __launch_bounds__(256, DIP_CAT_MINBLOCKS) k_cat_stats(CatArgs a, double* __restrict__ fwd, int VL, int PPB) {
  pdl_enter();
  const int v = threadIdx.x % VL, slot = threadIdx.x / VL;
  const CatLane l = cat_lane(a, v);
  const int w = a.W >> 1, nsrc = (a.H >> 1) * w;
  float4 acc[2] = {f4zero(), f4zero()};
  for (int p = slot < PPB ? blockIdx.x * PPB + slot : nsrc; p < nsrc; p += gridDim.x * PPB) {
    const int si = p / w, sj = p - si * w;
    float4 q[4];
    cat_quad<ACT>(a, l, si, sj, v, q);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      acc[0] = f4add(acc[0], q[e]);
      acc[1] = f4mla(q[e], q[e], acc[1]);
    }
  }
  double* const dst[2] = {fwd, fwd + (a.Cu + a.Cs) * kAccS};
  const int wid[2] = {a.Cu + a.Cs, a.Cu + a.Cs};
  block_reduce_atomic<2>(acc, VL, PPB, dst, wid);
}
void launch_cat_stats(CatArgs a, double* fwd_cat, int act_fun, cudaStream_t s) {
  VecGeom g = vec_geom(a.Cu + a.Cs, static_cast<long long>(a.H / 2) * (a.W / 2));
  auto kernel = act_pick(act_fun, [](auto x) { return k_cat_stats<decltype(x)::value>; });
  fit_grid(g, kernel, red_bytes(g, 2));
  launch_red(kernel, g.blocks, g.threads, red_bytes(g, 2), s, a, fwd_cat, g.VL, g.PPB);
}

// store the value of interior pixel (i, j) at its padded position and at every halo position that mirrors it
// (ZP: the border pixels of the image write the zeros of the halo cells next to them instead; the corner pixels also
// write the halo corner)
template <bool ZP = false>
__device__ __forceinline__ void store_with_halo(float* __restrict__ dst, int ld, int H, int W, int i, int j, int v, float4 val,
                                                Twin t16 = kNoTwin) {
  int rows[3], cols[3];
  int nr = 0, nc = 0;
  rows[nr++] = i + 1;
  if (i == (ZP ? 0 : 1)) rows[nr++] = 0;
  if (i == (ZP ? H - 1 : H - 2)) rows[nr++] = H + 1;
  cols[nc++] = j + 1;
  if (j == (ZP ? 0 : 1)) cols[nc++] = 0;
  if (j == (ZP ? W - 1 : W - 2)) cols[nc++] = W + 1;
  const int Wp = W + 2;
  for (int r = 0; r < nr; ++r)
    for (int c = 0; c < nc; ++c) {
      const float4 o = ZP && (r > 0 || c > 0) ? f4zero() : val;
      st4(dst + (static_cast<size_t>(rows[r]) * Wp + cols[c]) * ld + 4 * v, o);
      if (t16.p != nullptr) st4_bf16(t16.p + (static_cast<size_t>(rows[r]) * Wp + cols[c]) * t16.ld + 4 * v, o);
    }
}

template <bool ZP, int ACT>
__global__ void __launch_bounds__(256, DIP_CAT_MINBLOCKS) k_cat_write(CatArgs a, BnRef bn_cat, float* __restrict__ dst, int VL, int PPB, Twin t16) {
  pdl_enter();
  const int v = threadIdx.x % VL, slot = threadIdx.x / VL;
  const CatLane l = cat_lane(a, v);
  const Bn4 cf = bn_coef<0>(bn_cat, v);
  const int w = a.W >> 1, nsrc = (a.H >> 1) * w;
  const int ld = a.Cu + a.Cs;
  for (int p = slot < PPB ? blockIdx.x * PPB + slot : nsrc; p < nsrc; p += gridDim.x * PPB) {
    const int si = p / w, sj = p - si * w;
    float4 q[4];
    cat_quad<ACT>(a, l, si, sj, v, q);
#pragma unroll
    for (int e = 0; e < 4; ++e)
      store_with_halo<ZP>(dst, ld, a.H, a.W, 2 * si + (e >> 1), 2 * sj + (e & 1), v, bn_apply(cf, q[e]), t16);
  }
}
void launch_cat_write(CatArgs a, BnRef bn_cat, float* dst, int act_fun, cudaStream_t s, Twin t16, int zero_pad) {
  VecGeom g = vec_geom(a.Cu + a.Cs, static_cast<long long>(a.H / 2) * (a.W / 2));
  auto kernel = act_pick(act_fun, [&](auto x) {
    constexpr int A = decltype(x)::value;
    return zero_pad ? k_cat_write<true, A> : k_cat_write<false, A>;
  });
  fit_grid(g, kernel, 0);
  launch_k(kernel, dim3(g.blocks), dim3(g.threads), 0, s, 1, a, bn_cat, dst, g.VL, g.PPB, t16);
}

// ------------------------------------------------------------------------------------------------ gradient sources
// fold: adjoint of ReflectionPad2d(1). Interior (i,j) <- padded (i+1,j+1) plus mirrored halo rows/cols.
// ZP: adjoint of zero padding: the interior position only (the halo's gradient is dropped)
template <bool ZP = false>
__device__ __forceinline__ float4 fold_read(const float* __restrict__ gp, int ld, int coff, int H, int W, int i, int j,
                                            int v) {
  const int Wp = W + 2;
  const float* base = gp + coff + 4 * v;
  // the interior load is unconditional (issued at once, so several items' loads are in flight together); only the
  // one-pixel ring next to the border has mirrored halo positions to add
  float4 r = ld4(base + (static_cast<size_t>(i + 1) * Wp + (j + 1)) * ld);
  if (!ZP && (i == 1 || i == H - 2 || j == 1 || j == W - 2)) {
    int rows[3], cols[3];
    int nr = 0, nc = 0;
    rows[nr++] = i + 1;
    if (i == 1) rows[nr++] = 0;
    if (i == H - 2) rows[nr++] = H + 1;
    cols[nc++] = j + 1;
    if (j == 1) cols[nc++] = 0;
    if (j == W - 2) cols[nc++] = W + 1;
    for (int a = 0; a < nr; ++a)
      for (int b = 0; b < nc; ++b)
        if (a + b > 0) r = f4add(r, ld4(base + (static_cast<size_t>(rows[a]) * Wp + cols[b]) * ld));
  }
  return r;
}
// adjoint of x2 upsampling: D is [2H][2W][ld]
__device__ __forceinline__ float4 upadj_read(const float* __restrict__ D, int ld, int coff, int H, int W, int i, int j,
                                             int v, int bilinear) {
  const int H2 = 2 * H, W2 = 2 * W;
  float4 r = f4zero();
  const float* base = D + coff + 4 * v;
  if (!bilinear) {
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int b = 0; b < 2; ++b) r = f4add(r, ld4(base + (static_cast<size_t>(2 * i + a) * W2 + (2 * j + b)) * ld));
    return r;
  }
  const float wgt[4] = {0.25f, 0.75f, 0.75f, 0.25f};
  float4 t[16];
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const int y = min(max(2 * i - 1 + a, 0), H2 - 1);
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int x = min(max(2 * j - 1 + b, 0), W2 - 1);
      t[a * 4 + b] = ld4(base + (static_cast<size_t>(y) * W2 + x) * ld);
    }
  }
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) r = f4fma(wgt[a] * wgt[b], t[a * 4 + b], r);
  return r;
}
// per-thread constants of a gradient source
struct SrcRegs {
  float4 w[4];  // kind 1: skip-conv weight rows; kind 3: head weight rows
};
template <int KIND>
__device__ __forceinline__ SrcRegs src_regs(const GradSrc& s, int C, int v) {
  SrcRegs r;
#pragma unroll
  for (int k = 0; k < 4; ++k) r.w[k] = f4zero();
  if (KIND == 1 && s.ds != nullptr) {
    for (int k = 0; k < s.n2 && k < 4; ++k) r.w[k] = ld4(s.w2 + k * C + 4 * v);
  }
  if (KIND == 3) {
    for (int k = 0; k < s.nh && k < 4; ++k) r.w[k] = ld4(s.wh + k * C + 4 * v);
  }
  return r;
}
// gradient w.r.t. the BN(+act) output at pixel p = (i, j); dl (kind 3) returns the head's logit gradients
template <int KIND>
__device__ __forceinline__ float4 grad_read(const GradSrc& s, const SrcRegs& sr, int H, int W, int p, int i, int j, int v) {
  if (KIND == 0) return ld4(s.g + static_cast<size_t>(p) * s.ld + s.coff + 4 * v);
  if (KIND == 1) {
    float4 r = fold_read(s.g, s.ld, s.coff, H, W, i, j, v);
    if (s.ds != nullptr) {
      const float4 d = ld4(s.ds + static_cast<size_t>(p) * 4);  // n2 == 4
      r = f4fma(d.x, sr.w[0], r);
      r = f4fma(d.y, sr.w[1], r);
      r = f4fma(d.z, sr.w[2], r);
      r = f4fma(d.w, sr.w[3], r);
    }
    if (s.add != nullptr) r = f4add(r, ld4(s.add + static_cast<size_t>(p) * s.ld_add + 4 * v));
    return r;
  }
  if (KIND == 2) return upadj_read(s.g, s.ld, s.coff, H, W, i, j, v, s.bilinear);
  // KIND == 3: the item carries the 4 logit gradients of the pixel (k_head_dlogit); head_grad() expands them when consumed
  return ld4(s.dl4 + static_cast<size_t>(p) * 4);
}
// head source: gradient w.r.t. the last activation = sum_k dl[k] * w_head[k][c]
__device__ __forceinline__ float4 head_grad(const SrcRegs& sr, float4 d) {
  float4 r = f4zero();
  r = f4fma(d.x, sr.w[0], r);
  r = f4fma(d.y, sr.w[1], r);
  r = f4fma(d.z, sr.w[2], r);
  r = f4fma(d.w, sr.w[3], r);
  return r;
}

// Row-segment loop for kernels whose gradient source is a reflection-pad fold (padded dgrad output): a block takes units of
// (image row i, PPB * U consecutive pixels of that row), slot s handles pixels j0 + s + u * PPB.  One integer division per
// unit instead of one per pixel, row pointers hoisted, all loads of the unit issued before any is consumed, and the rare
// mirrored-halo additions (rows 1 / H-2, columns 1 / W-2) stay out of the load phase.  (The flat item_loop spent more
// than half of its instructions on index arithmetic here: 148 instructions per pixel vs 54 for a plain source.)
//   load(i, j, u) fills item u; use(i, j, u) consumes it; both are called with j < W only.
template <int U, class Load, class Use>
__device__ __forceinline__ void row_loop(int H, int W, int PPB, int slot, Load load, Use use) {
  const int seg = PPB * U, segs = (W + seg - 1) / seg;
  for (int unit = blockIdx.x; unit < H * segs; unit += gridDim.x) {
    const int i = unit / segs, j0 = (unit - i * segs) * seg + slot;
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (j0 + u * PPB < W) load(i, j0 + u * PPB, u);
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (j0 + u * PPB < W) use(i, j0 + u * PPB, u);
  }
}
// mirrored halo positions of interior pixel (i, j) added to its interior value r (fold = adjoint of ReflectionPad2d(1));
// ZP (adjoint of zero padding): nothing is added
template <bool ZP = false>
__device__ __forceinline__ float4 fold_border(const float* __restrict__ gp, int ld, int coff, int H, int W, int i, int j, int v,
                                              float4 r) {
  if (!ZP && (i == 1 || i == H - 2 || j == 1 || j == W - 2)) {
    const int Wp = W + 2;
    const float* base = gp + coff + 4 * v;
    const int r2 = i == 1 ? 0 : (i == H - 2 ? H + 1 : -1), c2 = j == 1 ? 0 : (j == W - 2 ? W + 1 : -1);
    if (r2 >= 0) r = f4add(r, ld4(base + (static_cast<size_t>(r2) * Wp + (j + 1)) * ld));
    if (c2 >= 0) r = f4add(r, ld4(base + (static_cast<size_t>(i + 1) * Wp + c2) * ld));
    if (r2 >= 0 && c2 >= 0) r = f4add(r, ld4(base + (static_cast<size_t>(r2) * Wp + c2) * ld));
    // an image of height (width) 3 has row (column) 1 == H-2: both mirrors apply
    if (i == 1 && i == H - 2) {
      r = f4add(r, ld4(base + (static_cast<size_t>(H + 1) * Wp + (j + 1)) * ld));
      if (c2 >= 0) r = f4add(r, ld4(base + (static_cast<size_t>(H + 1) * Wp + c2) * ld));
    }
    if (j == 1 && j == W - 2) {
      r = f4add(r, ld4(base + (static_cast<size_t>(i + 1) * Wp + (W + 1)) * ld));
      if (r2 >= 0) r = f4add(r, ld4(base + (static_cast<size_t>(r2) * Wp + (W + 1)) * ld));
      if (i == 1 && i == H - 2) r = f4add(r, ld4(base + (static_cast<size_t>(H + 1) * Wp + (W + 1)) * ld));
    }
  }
  return r;
}
struct FoldItem {
  float4 x, g, d;   // raw conv output; interior value of the padded gradient; skip-branch gradients (ds) or plain addend
};
__device__ __forceinline__ void fold_item_load(const GradSrc& s, const float* __restrict__ raw, int ld_raw, int W, int i, int j,
                                               int v, FoldItem& it) {
  const size_t p = static_cast<size_t>(i) * W + j;
  it.x = ld4(raw + p * ld_raw + 4 * v);
  it.g = ld4(s.g + s.coff + 4 * v + (static_cast<size_t>(i + 1) * (W + 2) + (j + 1)) * s.ld);
  if (s.ds != nullptr) it.d = ld4(s.ds + p * 4);
  else if (s.add != nullptr) it.d = ld4(s.add + p * s.ld_add + 4 * v);
}
template <bool ZP = false>
__device__ __forceinline__ float4 fold_item_grad(const GradSrc& s, const SrcRegs& sr, int H, int W, int i, int j, int v,
                                                 const FoldItem& it) {
  float4 r = fold_border<ZP>(s.g, s.ld, s.coff, H, W, i, j, v, it.g);
  if (s.ds != nullptr) {   // + the input gradient of the next level's 1x1 skip conv, computed on the fly
    r = f4fma(it.d.x, sr.w[0], r);
    r = f4fma(it.d.y, sr.w[1], r);
    r = f4fma(it.d.z, sr.w[2], r);
    r = f4fma(it.d.w, sr.w[3], r);
  } else if (s.add != nullptr) r = f4add(r, it.d);
  return r;
}

// ------------------------------------------------------------------------------------------------ BN(+LReLU) backward
struct RedItem {
  float4 x, g;  // raw conv output, gradient w.r.t. the BN(+act) output (head source: the pixel's logit gradients)
};
typedef RedItem BwdItem;
// dl4[p] = dout[k][p] * o[k][p] * (1 - o[k][p]) for k < K (else 0): sigmoid' folded into the logit gradient once per pixel
__global__ void k_head_dlogit(const float* __restrict__ dout, const float* __restrict__ outv, int K, int npix,
                              float* __restrict__ dl4, int sigmoid) {
  pdl_enter();
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < npix; p += gridDim.x * blockDim.x) {
    float d[4] = {0.f, 0.f, 0.f, 0.f};
    for (int k = 0; k < K; ++k) {
      const float o = outv[static_cast<size_t>(k) * npix + p];
      d[k] = dout[static_cast<size_t>(k) * npix + p] * (sigmoid ? o * (1.f - o) : 1.f);
    }
    st4(dl4 + static_cast<size_t>(p) * 4, make_float4(d[0], d[1], d[2], d[3]));
  }
}
void launch_head_dlogit(const float* dout, const float* outv, int K, int npix, float* dl4, cudaStream_t s, int sigmoid) {
  int blocks = (npix + 255) / 256;
  if (blocks > kNumSms * 8) blocks = kNumSms * 8;
  launch_k(k_head_dlogit, dim3(blocks), dim3(256), 0, s, 1, dout, outv, K, npix, dl4, sigmoid);
}

// ------------------------------------------------------------------------------------------------ input gradient
// NHWC -> NCHW transpose through a 32 x 32 shared tile (rows of 32 pixels of one image row x 32 channels), with the
// reflection-pad adjoint of the padded gradient and the skip-conv addend applied while reading (ZP: the zero-pad
// adjoint, the interior of the padded gradient only).
template <bool ZP>
__global__ void k_input_grad(const float* __restrict__ gp, const float* __restrict__ ds, int ld, int C, int H, int W,
                             float* __restrict__ dz) {
  pdl_enter();
  __shared__ float tile[32][33];
  const int i = blockIdx.y;
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int Wp = W + 2;
  for (int c0 = 0; c0 < C; c0 += 32) {
    for (int k = 0; k < 4; ++k) {
      const int j = blockIdx.x * 32 + ty + 8 * k, c = c0 + tx;
      float val = 0.f;
      if (j < W && c < C) {
        int rows[3], cols[3];
        int nr = 0, nc = 0;
        rows[nr++] = i + 1;
        if (!ZP && i == 1) rows[nr++] = 0;
        if (!ZP && i == H - 2) rows[nr++] = H + 1;
        cols[nc++] = j + 1;
        if (!ZP && j == 1) cols[nc++] = 0;
        if (!ZP && j == W - 2) cols[nc++] = W + 1;
        for (int a = 0; a < nr; ++a)
          for (int b = 0; b < nc; ++b) val += gp[(static_cast<size_t>(rows[a]) * Wp + cols[b]) * ld + c];
        if (ds != nullptr) val += ds[(static_cast<size_t>(i) * W + j) * ld + c];
      }
      tile[ty + 8 * k][tx] = val;   // [pixel][channel]
    }
    __syncthreads();
    for (int k = 0; k < 4; ++k) {
      const int c = c0 + ty + 8 * k, j = blockIdx.x * 32 + tx;
      if (j < W && c < C) dz[(static_cast<size_t>(c) * H + i) * W + j] = tile[tx][ty + 8 * k];
    }
    __syncthreads();
  }
}
void launch_input_grad(const float* gp, const float* ds, int ld, int C, int H, int W, float* dz, cudaStream_t s, int zero_pad) {
  dim3 grid((W + 31) / 32, H), block(32, 8);
  launch_k(zero_pad ? k_input_grad<true> : k_input_grad<false>, dim3(grid), dim3(block), 0, s, 1, gp, ds, ld, C, H, W, dz);
}
// ZP applies to KIND 1 only: the padded gradient's halo is dropped instead of folded (zero-padding adjoint).
// ACT: the activation's adjoint (act != 0), from the pre-activation recomputed from raw, as in the forward.
template <int KIND, bool ZP = false, int ACT = kActLeakyRelu>
__device__ __forceinline__ void d_bn_bwd_reduce(const float* __restrict__ raw, int ld_raw, BnRef bn, int act, GradSrc src,
                                                       int H, int W, double* __restrict__ bwd, int VL, int PPB) {
  const int v = threadIdx.x % VL, slot = threadIdx.x / VL;
  const Bn4 cf = bn_coef<0>(bn, v);
  const SrcRegs sr = src_regs<KIND>(src, bn.C, v);
  float4 acc[2] = {f4zero(), f4zero()};
  if constexpr (KIND == 1) {
    FoldItem it[DIP_U_BWD1];
    row_loop<DIP_U_BWD1>(H, W, PPB, slot,
                         [&](int i, int j, int u) { fold_item_load(src, raw, ld_raw, W, i, j, v, it[u]); },
                         [&](int i, int j, int u) {
                           float4 dz = fold_item_grad<ZP>(src, sr, H, W, i, j, v, it[u]);
                           if (act) dz = act_bwd4<ACT>(bn_apply(cf, it[u].x), dz);
                           acc[0] = f4add(acc[0], dz);
                           acc[1] = f4mla(dz, bn_xhat(cf, it[u].x), acc[1]);
                         });
  } else
  item_loop<KIND == 3 ? 8 : (KIND == 0 ? 4 : (KIND == 1 ? DIP_U_BWD1 : 2))>(
      blockIdx.x * PPB + slot, gridDim.x * PPB, H * W,
      [&](int p) {
        RedItem it;
        const int i = p / W, j = p - i * W;
        it.x = ld4(raw + static_cast<size_t>(p) * ld_raw + 4 * v);
        it.g = grad_read<KIND>(src, sr, H, W, p, i, j, v);
        return it;
      },
      [&](int, const RedItem& it) {
        float4 dz = KIND == 3 ? head_grad(sr, it.g) : it.g;
        if (act) dz = act_bwd4<ACT>(bn_apply(cf, it.x), dz);
        acc[0] = f4add(acc[0], dz);
        acc[1] = f4mla(dz, bn_xhat(cf, it.x), acc[1]);
      });
  double* const dst[2] = {bwd, bwd + bn.C * kAccS};
  const int wid[2] = {bn.C, bn.C};
  block_reduce_atomic<2>(acc, VL, PPB, dst, wid);
}
template <int KIND, bool ZP = false, int ACT = kActLeakyRelu>
__global__ void __launch_bounds__(256, (KIND == 0 || KIND == 2) ? 3 : 2) k_bn_bwd_reduce(const float* __restrict__ raw, int ld_raw, BnRef bn, int act, GradSrc src,
                                                       int H, int W, double* __restrict__ bwd, int VL, int PPB) {
  pdl_enter();
  d_bn_bwd_reduce<KIND, ZP, ACT>(raw, ld_raw, bn, act, src, H, W, bwd, VL, PPB);
}
void launch_bn_bwd_reduce(const float* raw, int ld_raw, BnRef bn, int act, int act_fun, GradSrc src, int H, int W,
                          double* bwd, cudaStream_t s) {
  VecGeom g = vec_geom(bn.C, static_cast<long long>(H) * W);
  const size_t sm = red_bytes(g, 2);
  auto kernel = act_pick(act_fun, [&](auto a) {
    constexpr int A = decltype(a)::value;
    return src.kind == 0 ? k_bn_bwd_reduce<0, false, A>
         : src.kind == 1 ? (src.zero_pad ? k_bn_bwd_reduce<1, true, A> : k_bn_bwd_reduce<1, false, A>)
         : src.kind == 2 ? k_bn_bwd_reduce<2, false, A> : k_bn_bwd_reduce<3, false, A>;
  });
  fit_grid(g, kernel, sm);
  launch_red(kernel, g.blocks, g.threads, sm, s, raw, ld_raw, bn, act, src, H, W, bwd, g.VL, g.PPB);
}

// apply pass; for the head source (KIND 3) it also accumulates the head's own gradients:
//   dW_head[k][c] += dl[k] * act(bn(raw))[c],  db_head[k] += dl[k]
template <int KIND, bool ZP = false, int ACT = kActLeakyRelu>
__global__ void __launch_bounds__(256, KIND == 2 ? 3 : 2) k_bn_bwd_apply(const float* __restrict__ raw, int ld_raw, BnRef bn, int act, GradSrc src,
                                                      int H, int W, const double* __restrict__ bwd, float* __restrict__ draw,
                                                      double* __restrict__ dbias, int VL, int PPB, Twin t16) {
  pdl_enter();
  const int v = threadIdx.x % VL, slot = threadIdx.x / VL;
  const Bn4 cf = bn_coef<0>(bn, v);
  const SrcRegs sr = src_regs<KIND>(src, bn.C, v);
  const int C = bn.C;
  float4 m1, m2;
  bwd_means<0>(bwd, C, bn.inv_n, v, m1, m2);
  constexpr int K = KIND == 3 ? 6 : 1;
  float4 acc[K];
#pragma unroll
  for (int k = 0; k < K; ++k) acc[k] = f4zero();
  if constexpr (KIND == 1) {
    FoldItem it[DIP_U_BWD1];
    row_loop<DIP_U_BWD1>(H, W, PPB, slot,
                         [&](int i, int j, int u) { fold_item_load(src, raw, ld_raw, W, i, j, v, it[u]); },
                         [&](int i, int j, int u) {
                           float4 dz = fold_item_grad<ZP>(src, sr, H, W, i, j, v, it[u]);
                           if (act) dz = act_bwd4<ACT>(bn_apply(cf, it[u].x), dz);
                           const float4 xh = bn_xhat(cf, it[u].x);
                           float4 dx;
                           dx.x = cf.scale.x * (dz.x - m1.x - xh.x * m2.x);
                           dx.y = cf.scale.y * (dz.y - m1.y - xh.y * m2.y);
                           dx.z = cf.scale.z * (dz.z - m1.z - xh.z * m2.z);
                           dx.w = cf.scale.w * (dz.w - m1.w - xh.w * m2.w);
                           if (draw != nullptr) st4(draw + (static_cast<size_t>(i) * W + j) * C + 4 * v, dx);
                           if (t16.p != nullptr) st4_bf16(t16.p + (static_cast<size_t>(i) * W + j) * t16.ld + 4 * v, dx);
                           acc[0] = f4add(acc[0], dx);
                         });
  } else
  item_loop<(KIND == 0 || KIND == 3) ? 4 : (KIND == 1 ? DIP_U_BWD1 : 2)>(
      blockIdx.x * PPB + slot, gridDim.x * PPB, H * W,
      [&](int p) {
        BwdItem it;
        const int i = p / W, j = p - i * W;
        it.x = ld4(raw + static_cast<size_t>(p) * ld_raw + 4 * v);
        it.g = grad_read<KIND>(src, sr, H, W, p, i, j, v);
        return it;
      },
      [&](int p, const BwdItem& it) {
        float4 dz = KIND == 3 ? head_grad(sr, it.g) : it.g;
        const float4 y = bn_apply(cf, it.x);
        if constexpr (KIND == 3) {
          const float4 u = act ? act_fwd4<ACT>(y) : y;
#pragma unroll
          acc[1] = f4fma(it.g.x, u, acc[1]);
          acc[2] = f4fma(it.g.y, u, acc[2]);
          acc[3] = f4fma(it.g.z, u, acc[3]);
          acc[4] = f4fma(it.g.w, u, acc[4]);
          if (v == 0) acc[5] = f4add(acc[5], it.g);
        }
        if (act) dz = act_bwd4<ACT>(y, dz);
        const float4 xh = bn_xhat(cf, it.x);
        float4 dx;
        dx.x = cf.scale.x * (dz.x - m1.x - xh.x * m2.x);
        dx.y = cf.scale.y * (dz.y - m1.y - xh.y * m2.y);
        dx.z = cf.scale.z * (dz.z - m1.z - xh.z * m2.z);
        dx.w = cf.scale.w * (dz.w - m1.w - xh.w * m2.w);
        if (draw != nullptr) st4(draw + static_cast<size_t>(p) * C + 4 * v, dx);
        if (t16.p != nullptr) st4_bf16(t16.p + static_cast<size_t>(p) * t16.ld + 4 * v, dx);
        acc[0] = f4add(acc[0], dx);
      });
  if constexpr (KIND == 3) {
    double* const dst[K] = {dbias, src.dwh, src.nh > 1 ? src.dwh + C * kAccS : nullptr,
                            src.nh > 2 ? src.dwh + 2 * C * kAccS : nullptr, src.nh > 3 ? src.dwh + 3 * C * kAccS : nullptr, src.dbh};
    // acc[5] (db_head) is non-zero on lanes v == 0 only: its 4 leading "channels" are the per-output bias gradients
    const int wid[K] = {C, C, C, C, C, src.nh};
    block_reduce_atomic<K>(acc, VL, PPB, dst, wid);
  } else {
    double* const dst[1] = {dbias};
    const int wid[1] = {C};
    block_reduce_atomic<K>(acc, VL, PPB, dst, wid);
  }
}
void launch_bn_bwd_apply(const float* raw, int ld_raw, BnRef bn, int act, int act_fun, GradSrc src, int H, int W,
                         const double* bwd, float* draw, double* dbias, cudaStream_t s, Twin t16) {
  VecGeom g = vec_geom(bn.C, static_cast<long long>(H) * W);
  const size_t sm = red_bytes(g, src.kind == 3 ? 6 : 1);
  auto kernel = act_pick(act_fun, [&](auto a) {
    constexpr int A = decltype(a)::value;
    return src.kind == 0 ? k_bn_bwd_apply<0, false, A>
         : src.kind == 1 ? (src.zero_pad ? k_bn_bwd_apply<1, true, A> : k_bn_bwd_apply<1, false, A>)
         : src.kind == 2 ? k_bn_bwd_apply<2, false, A> : k_bn_bwd_apply<3, false, A>;
  });
  fit_grid(g, kernel, sm);
  launch_red(kernel, g.blocks, g.threads, sm, s, raw, ld_raw, bn, act, src, H, W, bwd, draw, dbias, g.VL, g.PPB, t16);
}

// ------------------------------------------------------------------------------------------------ concat-BN backward
// The concat BN has no activation behind it, and its output y = gamma * xhat + beta is still in HBM (the padded conv
// input P_cat), so xhat = (y - beta) / gamma is recovered from the stored tensor instead of re-running the upsampling.
// (gamma == 0 exactly: xhat is taken as 0; dx is 0 in that case anyway.)
struct CatBwdCoef {
  float4 beta, inv_gamma, scale;
};
__device__ __forceinline__ CatBwdCoef cat_bwd_coef(const BnRef& bn, int v) {
  __shared__ __align__(16) float s_beta[kMaxBnC], s_ig[kMaxBnC], s_sc[kMaxBnC];
  for (int c = threadIdx.x; c < bn.C; c += blockDim.x) {
    const int ct = (c + bn.rot) % bn.C;
    const double m = acc_get(bn.fwd + c * kAccS) * static_cast<double>(bn.inv_n);
    double var = acc_get(bn.fwd + (bn.C + c) * kAccS) * static_cast<double>(bn.inv_n) - m * m;
    if (var < 0.0) var = 0.0;
    const float g = bn.gamma[ct];
    s_beta[c] = bn.beta[ct];
    s_ig[c] = g != 0.f ? 1.f / g : 0.f;
    s_sc[c] = g * static_cast<float>(1.0 / sqrt(var + static_cast<double>(kBnEps)));
  }
  __syncthreads();
  CatBwdCoef r;
  r.beta = *reinterpret_cast<const float4*>(&s_beta[4 * v]);
  r.inv_gamma = *reinterpret_cast<const float4*>(&s_ig[4 * v]);
  r.scale = *reinterpret_cast<const float4*>(&s_sc[4 * v]);
  return r;
}
__device__ __forceinline__ float4 cat_xhat(const CatBwdCoef& c, float4 y) {
  return make_float4((y.x - c.beta.x) * c.inv_gamma.x, (y.y - c.beta.y) * c.inv_gamma.y, (y.z - c.beta.z) * c.inv_gamma.z,
                     (y.w - c.beta.w) * c.inv_gamma.w);
}
template <bool ZP>
__global__ void __launch_bounds__(256) k_cat_bwd_reduce(const float* __restrict__ pcat, BnRef bn_cat, const float* __restrict__ gp,
                                                        int ld, int H, int W, double* __restrict__ bwd, int VL, int PPB) {
  pdl_enter();
  const int v = threadIdx.x % VL, slot = threadIdx.x / VL;
  const CatBwdCoef cf = cat_bwd_coef(bn_cat, v);
  const int Wp = W + 2;
  float4 acc[2] = {f4zero(), f4zero()};
  // (no row-segment loop as in the BN backward kernels: with 33 lanes per pixel a unit would be only 14 pixels)
  item_loop<DIP_U_CATBWD>(slot < PPB ? blockIdx.x * PPB + slot : H * W, gridDim.x * PPB, H * W,
               [&](int p) {
                 RedItem it;
                 const int i = p / W, j = p - i * W;
                 it.x = ld4(pcat + (static_cast<size_t>(i + 1) * Wp + (j + 1)) * ld + 4 * v);
                 it.g = fold_read<ZP>(gp, ld, 0, H, W, i, j, v);
                 return it;
               },
               [&](int, const RedItem& it) {
                 acc[0] = f4add(acc[0], it.g);
                 acc[1] = f4mla(it.g, cat_xhat(cf, it.x), acc[1]);
               });
  double* const dst[2] = {bwd, bwd + bn_cat.C * kAccS};
  const int wid[2] = {bn_cat.C, bn_cat.C};
  block_reduce_atomic<2>(acc, VL, PPB, dst, wid);
}
void launch_cat_bwd_reduce(const float* pcat, BnRef bn_cat, const float* gp, int ld, int H, int W, double* bwd,
                           cudaStream_t s, int zero_pad) {
  VecGeom g = vec_geom(bn_cat.C, static_cast<long long>(H) * W);
  auto kernel = zero_pad ? k_cat_bwd_reduce<true> : k_cat_bwd_reduce<false>;
  fit_grid(g, kernel, red_bytes(g, 2));
  launch_red(kernel, g.blocks, g.threads, red_bytes(g, 2), s, pcat, bn_cat, gp, ld, H, W, bwd, g.VL, g.PPB);
}
template <bool ZP>
__global__ void __launch_bounds__(256) k_cat_bwd_apply(const float* __restrict__ pcat, BnRef bn_cat, const float* __restrict__ gp,
                                                       int ld, int H, int W, const double* __restrict__ bwd,
                                                       float* __restrict__ dcat, int VL, int PPB) {
  pdl_enter();
  const int v = threadIdx.x % VL, slot = threadIdx.x / VL;
  const CatBwdCoef cf = cat_bwd_coef(bn_cat, v);
  const int C = bn_cat.C;
  const int Wp = W + 2;
  float4 m1, m2;
  bwd_means<0>(bwd, C, bn_cat.inv_n, v, m1, m2);
  item_loop<DIP_U_CATBWD>(slot < PPB ? blockIdx.x * PPB + slot : H * W, gridDim.x * PPB, H * W,
               [&](int p) {
                 RedItem it;
                 const int i = p / W, j = p - i * W;
                 it.x = ld4(pcat + (static_cast<size_t>(i + 1) * Wp + (j + 1)) * ld + 4 * v);
                 it.g = fold_read<ZP>(gp, ld, 0, H, W, i, j, v);
                 return it;
               },
               [&](int p, const RedItem& it) {
                 const float4 xh = cat_xhat(cf, it.x);
                 float4 dx;
                 dx.x = cf.scale.x * (it.g.x - m1.x - xh.x * m2.x);
                 dx.y = cf.scale.y * (it.g.y - m1.y - xh.y * m2.y);
                 dx.z = cf.scale.z * (it.g.z - m1.z - xh.z * m2.z);
                 dx.w = cf.scale.w * (it.g.w - m1.w - xh.w * m2.w);
                 st4(dcat + static_cast<size_t>(p) * C + 4 * v, dx);
               });
}
void launch_cat_bwd_apply(const float* pcat, BnRef bn_cat, const float* gp, int ld, int H, int W, const double* bwd,
                          float* dcat, cudaStream_t s, int zero_pad) {
  VecGeom g = vec_geom(bn_cat.C, static_cast<long long>(H) * W);
  auto kernel = zero_pad ? k_cat_bwd_apply<true> : k_cat_bwd_apply<false>;
  fit_grid(g, kernel, 0);
  launch_k(kernel, dim3(g.blocks), dim3(g.threads), 0, s, 1, pcat, bn_cat, gp, ld, H, W, bwd, dcat, g.VL, g.PPB);
}

// Adjoint of the x2 upsampling, materialised once: dst[h][w][C] <- D[2h][2w][ld] (channels coff..coff+C)
__global__ void __launch_bounds__(256) k_upadj(const float* __restrict__ D, int ld, int coff, int h, int w, int C, int bilinear,
                                               float* __restrict__ dst, int VL, int PPB) {
  pdl_enter();
  const int v = threadIdx.x % VL, slot = threadIdx.x / VL;
  item_loop<1>(blockIdx.x * PPB + slot, gridDim.x * PPB, h * w,
               [&](int p) {
                 const int i = p / w, j = p - i * w;
                 return upadj_read(D, ld, coff, h, w, i, j, v, bilinear);
               },
               [&](int p, float4 g) { st4(dst + static_cast<size_t>(p) * C + 4 * v, g); });
}
void launch_upadj(const float* D, int ld, int coff, int h, int w, int C, int bilinear, float* dst, cudaStream_t s) {
  VecGeom g = vec_geom(C, static_cast<long long>(h) * w);
  fit_grid(g, k_upadj, 0);
  launch_k(k_upadj, dim3(g.blocks), dim3(g.threads), 0, s, 1, D, ld, coff, h, w, C, bilinear, dst, g.VL, g.PPB);
}

// ------------------------------------------------------------------------------------------------ 2 x 2 average pooling
__global__ void __launch_bounds__(256) k_avgpool2(const float* __restrict__ x, int h, int w, int C, float* __restrict__ y, int VL, int PPB) {
  pdl_enter();
  const int v = threadIdx.x % VL, slot = threadIdx.x / VL;
  const int W2 = 2 * w;
  item_loop<2>(blockIdx.x * PPB + slot, gridDim.x * PPB, h * w,
               [&](int p) {
                 const int i = p / w, j = p - i * w;
                 const float* b = x + (static_cast<size_t>(2 * i) * W2 + 2 * j) * C + 4 * v;
                 const float4 a0 = ld4(b), a1 = ld4(b + C), a2 = ld4(b + static_cast<size_t>(W2) * C), a3 = ld4(b + static_cast<size_t>(W2 + 1) * C);
                 return f4add(f4add(a0, a1), f4add(a2, a3));
               },
               [&](int p, float4 t) { st4(y + static_cast<size_t>(p) * C + 4 * v, make_float4(0.25f * t.x, 0.25f * t.y, 0.25f * t.z, 0.25f * t.w)); });
}
void launch_avgpool2(const float* x, int h, int w, int C, float* y, cudaStream_t s) {
  VecGeom g = vec_geom(C, static_cast<long long>(h) * w);
  fit_grid(g, k_avgpool2, 0);
  launch_k(k_avgpool2, dim3(g.blocks), dim3(g.threads), 0, s, 1, x, h, w, C, y, g.VL, g.PPB);
}
__global__ void __launch_bounds__(256) k_avgpool2_bwd(const float* __restrict__ dy, int h, int w, int C, float* __restrict__ dx, int VL,
                                                      int PPB, Twin t16) {
  pdl_enter();
  const int v = threadIdx.x % VL, slot = threadIdx.x / VL;
  const int W2 = 2 * w;
  item_loop<2>(blockIdx.x * PPB + slot, gridDim.x * PPB, h * w,
               [&](int p) { return ld4(dy + static_cast<size_t>(p) * C + 4 * v); },
               [&](int p, float4 t) {
                 const int i = p / w, j = p - i * w;
                 const float4 q = make_float4(0.25f * t.x, 0.25f * t.y, 0.25f * t.z, 0.25f * t.w);
#pragma unroll
                 for (int a = 0; a < 4; ++a) {
                   const size_t o = static_cast<size_t>(2 * i + (a >> 1)) * W2 + 2 * j + (a & 1);
                   if (dx != nullptr) st4(dx + o * C + 4 * v, q);
                   if (t16.p != nullptr) st4_bf16(t16.p + o * t16.ld + 4 * v, q);
                 }
               });
}
void launch_avgpool2_bwd(const float* dy, int h, int w, int C, float* dx, cudaStream_t s, Twin t16) {
  VecGeom g = vec_geom(C, static_cast<long long>(h) * w);
  fit_grid(g, k_avgpool2_bwd, 0);
  launch_k(k_avgpool2_bwd, dim3(g.blocks), dim3(g.threads), 0, s, 1, dy, h, w, C, dx, g.VL, g.PPB, t16);
}

// weight row n of a skinny conv for lanes 4v..4v+3: rows are cw long (cw < C when the stored depth is zero-padded)
__device__ __forceinline__ float4 skinny_wrow(const float* __restrict__ w, int n, int cw, int v) {
  if ((cw & 3) == 0) return 4 * v < cw ? ld4(w + n * cw + 4 * v) : f4zero();
  const float* r = w + n * cw;
  const int c = 4 * v;
  return make_float4(c < cw ? r[c] : 0.f, c + 1 < cw ? r[c + 1] : 0.f, c + 2 < cw ? r[c + 2] : 0.f, c + 3 < cw ? r[c + 3] : 0.f);
}

// ------------------------------------------------------------------------------------------------ skinny 1x1 convs
// VL = C/4 lanes per pixel, rounded up to a power of two VLp <= 32 so that a pixel's lanes are an aligned group of the warp
// for the shuffle reduction (C = 24, 40, 48, ... : VL = 6, 10, 12, ...); lanes v >= VL hold zeros.
__host__ __device__ __forceinline__ int skinny_lanes(int C) {
  int vlp = 1;
  while (vlp < C / 4) vlp <<= 1;
  return vlp;
}
__device__ __forceinline__ void d_skinny_fwd_narrow(const float* __restrict__ x, int ldx, int x_rs, const float* __restrict__ w,
                                                    const float* __restrict__ b, int C, int N, int H, int W,
                                                    float* __restrict__ y, int mode, double* __restrict__ stats, int cw) {
  const int VL = C / 4, VLp = skinny_lanes(C);
  const int PPB = 256 / VLp;
  const int v = threadIdx.x % VLp, slot = threadIdx.x / VLp;
  const int npix = H * W;
  float4 wv[4];
  float bv[4];
#pragma unroll
  for (int n = 0; n < 4; ++n) {
    wv[n] = n < N ? skinny_wrow(w, n, cw, v) : f4zero();
    bv[n] = (n < N && b != nullptr) ? b[n] : 0.f;
  }
  float4 s1 = f4zero(), s2 = f4zero();
  // every thread runs the same number of trips so that the shuffles stay warp-convergent
  const int trips = (npix + gridDim.x * PPB - 1) / (gridDim.x * PPB);
  for (int t = 0; t < trips; ++t) {
    const int p = (t * gridDim.x + blockIdx.x) * PPB + slot;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    if (p < npix && v < VL) {
      const int i = p / W, j = p - i * W;
      const float4 xv = ld4(x + (static_cast<size_t>(i) * x_rs + j) * ldx + 4 * v);
#pragma unroll
      for (int n = 0; n < 4; ++n) acc[n] = f4dot(xv, wv[n]);
    }
    for (int o = VLp >> 1; o > 0; o >>= 1) {
#pragma unroll
      for (int n = 0; n < 4; ++n) acc[n] += __shfl_xor_sync(0xffffffffu, acc[n], o);
    }
    if (p < npix && v == 0) {
      float o4[4];
#pragma unroll
      for (int n = 0; n < 4; ++n) o4[n] = n < N ? acc[n] + bv[n] : 0.f;
      if (mode == 0) {
        if (N == 4) st4(y + static_cast<size_t>(p) * 4, make_float4(o4[0], o4[1], o4[2], o4[3]));
        else for (int n = 0; n < N; ++n) y[static_cast<size_t>(p) * N + n] = o4[n];
        const float4 ov = make_float4(o4[0], o4[1], o4[2], o4[3]);
        s1 = f4add(s1, ov);
        s2 = f4mla(ov, ov, s2);
      } else {
        for (int n = 0; n < N; ++n) y[static_cast<size_t>(n) * npix + p] = (mode == 1) ? 1.f / (1.f + expf(-o4[n])) : o4[n];
      }
    }
  }
  if (stats != nullptr) {
    // only lanes v == 0 hold data; treat every thread as a slot of one 4-channel group (VL = 1)
    float4 acc2[2] = {s1, s2};
    double* const dst[2] = {stats, stats + N * kAccS};
    const int wid[2] = {N, N};
    block_reduce_atomic<2>(acc2, 1, 256, dst, wid);
  }
}
// Wide inputs (G = C/4 = 8, 16 or 32 lanes per pixel): a lane group takes U = G/4 CONSECUTIVE pixels per trip, forms the
// 4 x U partial dot products of its 4 channels, and all 4U = G values are reduced over the group with a value-halving butterfly
// (G - 1 shuffles per U pixels instead of 4 * log2(G) per pixel: 7 vs 24 for C = 32, 31 vs 160 for C = 128).  Afterwards lane l
// of the group holds output n = l / U of pixel u = l % U, so a group's 4U outputs are 4U consecutive floats of y.
template <int G>
__device__ __forceinline__ void d_skinny_fwd_wide(const float* __restrict__ x, int ldx, int x_rs, const float* __restrict__ w,
                                                  const float* __restrict__ b, int N, int H, int W, float* __restrict__ y,
                                                  double* __restrict__ stats, int cw) {
  constexpr int U = G / 4;
  const int v = threadIdx.x % G, grp = threadIdx.x / G;
  const int groups = blockDim.x / G;                 // groups per block; a block covers groups * U = 64 pixels per trip
  const int npix = H * W;
  float4 wv[4];
#pragma unroll
  for (int n = 0; n < 4; ++n) wv[n] = n < N ? skinny_wrow(w, n, cw, v) : f4zero();
  const int my_n = v / U, my_u = v % U;              // what this lane owns after the butterfly
  const float my_b = (my_n < N && b != nullptr) ? b[my_n] : 0.f;
  float s1 = 0.f, s2 = 0.f;
  const int per_trip = gridDim.x * groups * U;
  const int trips = (npix + per_trip - 1) / per_trip;   // the same for every thread: the shuffles stay warp-convergent
  for (int t = 0; t < trips; ++t) {
    const int p0 = ((t * gridDim.x + blockIdx.x) * groups + grp) * U;
    float4 xv[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int p = p0 + u;
      xv[u] = f4zero();
      if (p < npix) {
        const int i = p / W, j = p - i * W;
        xv[u] = ld4(x + (static_cast<size_t>(i) * x_rs + j) * ldx + 4 * v);
      }
    }
    float vals[4 * U];
#pragma unroll
    for (int n = 0; n < 4; ++n)
#pragma unroll
      for (int u = 0; u < U; ++u) vals[n * U + u] = f4dot(xv[u], wv[n]);
    // value-halving butterfly: after the step with offset o, a lane keeps the half of its values selected by its bit o
#pragma unroll
    for (int o = G / 2, cnt = 2 * U; o >= 1; o >>= 1, cnt >>= 1) {   // cnt = values kept after this step
      const bool up = (v & o) != 0;
#pragma unroll
      for (int k = 0; k < cnt; ++k) {
        const float lo = vals[k], hi = vals[k + cnt];
        vals[k] = (up ? hi : lo) + __shfl_xor_sync(0xffffffffu, up ? lo : hi, o);
      }
    }
    const int p = p0 + my_u;
    if (p < npix && my_n < N) {
      const float o = vals[0] + my_b;
      y[static_cast<size_t>(p) * N + my_n] = o;
      s1 += o;
      s2 = fmaf(o, o, s2);
    }
  }
  if (stats != nullptr) {
    float4 acc2[2] = {f4zero(), f4zero()};
    float* a1 = reinterpret_cast<float*>(&acc2[0]);
    float* a2 = reinterpret_cast<float*>(&acc2[1]);
#pragma unroll
    for (int n = 0; n < 4; ++n) { a1[n] = my_n == n ? s1 : 0.f; a2[n] = my_n == n ? s2 : 0.f; }
    double* const dst[2] = {stats, stats + N * kAccS};
    const int wid[2] = {N, N};
    block_reduce_atomic<2>(acc2, 1, 256, dst, wid);
  }
}
__global__ void __launch_bounds__(256) k_skinny_fwd(const float* __restrict__ x, int ldx, int x_rs, const float* __restrict__ w,
                                                    const float* __restrict__ b, int C, int N, int H, int W,
                                                    float* __restrict__ y, int mode, double* __restrict__ stats, int cw) {
  pdl_enter();
  if (mode == 0 && C == 128) d_skinny_fwd_wide<32>(x, ldx, x_rs, w, b, N, H, W, y, stats, cw);
  else if (mode == 0 && C == 64) d_skinny_fwd_wide<16>(x, ldx, x_rs, w, b, N, H, W, y, stats, cw);
  else if (mode == 0 && C == 32) d_skinny_fwd_wide<8>(x, ldx, x_rs, w, b, N, H, W, y, stats, cw);
  else d_skinny_fwd_narrow(x, ldx, x_rs, w, b, C, N, H, W, y, mode, stats, cw);
}
void launch_skinny_fwd(const float* x, int ldx, int x_rs, const float* w, const float* b, int C, int N, int H,
                       int W, float* y, int mode, double* stats, cudaStream_t s, int cw) {
  const bool wide = mode == 0 && (C == 32 || C == 64 || C == 128);
  const int PPB = wide ? 64 : 256 / skinny_lanes(C);   // pixels per block and trip of the path k_skinny_fwd takes
  long long nb = (static_cast<long long>(H) * W + PPB - 1) / PPB;
  if (nb > kNumSms * 8) nb = kNumSms * 8;
  launch_red(k_skinny_fwd, static_cast<int>(nb), 256, 2 * 256 * sizeof(float4) + 2 * 4 * sizeof(double), s, x, ldx, x_rs, w, b, C, N, H, W,
                  y, mode, stats, cw > 0 ? cw : C);
}

__global__ void k_skinny_bwd(const float* __restrict__ x, int ldx, int x_rs, const float* __restrict__ w, int C, int N,
                             int H, int W, const float* __restrict__ dy, const float* __restrict__ out_nchw, int mode,
                             float* __restrict__ dx, double* __restrict__ dw, double* __restrict__ db, int VL, int PPB, int cw) {
  pdl_enter();
  const int v = threadIdx.x % VL, slot = threadIdx.x / VL;
  const int npix = H * W;
  float4 wv[4];
  for (int n = 0; n < 4; ++n) wv[n] = n < N ? skinny_wrow(w, n, cw, v) : f4zero();
  float4 acc[5] = {f4zero(), f4zero(), f4zero(), f4zero(), f4zero()};  // dw rows 0..3, db (lane v == 0 only)
  struct Item { float4 g, x; };
  item_loop<4>(blockIdx.x * PPB + slot, gridDim.x * PPB, npix,
               [&](int p) {
                 Item it;
                 const int i = p / W, j = p - i * W;
                 float g[4] = {0.f, 0.f, 0.f, 0.f};
                 if (mode == 0 && N == 4) {
                   it.g = ld4(dy + static_cast<size_t>(p) * 4);
                 } else {
                   for (int n = 0; n < N; ++n) {
                     if (mode == 0) g[n] = dy[static_cast<size_t>(p) * N + n];
                     else {
                       const float d = dy[static_cast<size_t>(n) * npix + p];
                       if (mode == 1) { const float o = out_nchw[static_cast<size_t>(n) * npix + p]; g[n] = d * o * (1.f - o); } else g[n] = d;
                     }
                   }
                   it.g = make_float4(g[0], g[1], g[2], g[3]);
                 }
                 it.x = ld4(x + (static_cast<size_t>(i) * x_rs + j) * ldx + 4 * v);
                 return it;
               },
               [&](int p, const Item& it) {
                 acc[0] = f4fma(it.g.x, it.x, acc[0]);
                 acc[1] = f4fma(it.g.y, it.x, acc[1]);
                 acc[2] = f4fma(it.g.z, it.x, acc[2]);
                 acc[3] = f4fma(it.g.w, it.x, acc[3]);
                 if (v == 0) acc[4] = f4add(acc[4], it.g);
                 if (dx != nullptr) {
                   float4 d = f4zero();
                   d = f4fma(it.g.x, wv[0], d);
                   d = f4fma(it.g.y, wv[1], d);
                   d = f4fma(it.g.z, wv[2], d);
                   d = f4fma(it.g.w, wv[3], d);
                   st4(dx + static_cast<size_t>(p) * C + 4 * v, d);
                 }
               });
  double* const dst[5] = {dw, N > 1 ? dw + C * kAccS : nullptr, N > 2 ? dw + 2 * C * kAccS : nullptr,
                          N > 3 ? dw + 3 * C * kAccS : nullptr, db};
  const int wid[5] = {C, C, C, C, N};  // acc[4] (bias gradient) lives on lanes v == 0 only
  block_reduce_atomic<5>(acc, VL, PPB, dst, wid);
}
void launch_skinny_bwd(const float* x, int ldx, int x_rs, const float* w, int C, int N, int H, int W,
                       const float* dy, const float* out_nchw, int mode, float* dx, double* dw, double* db,
                       cudaStream_t s, int cw) {
  VecGeom g = vec_geom(C, static_cast<long long>(H) * W);
  fit_grid(g, k_skinny_bwd, red_bytes(g, 5));
  launch_red(k_skinny_bwd, g.blocks, g.threads, red_bytes(g, 5), s, x, ldx, x_rs, w, C, N, H, W, dy, out_nchw, mode, dx, dw, db,
                                                             g.VL, g.PPB, cw > 0 ? cw : C);
}

// ------------------------------------------------------------------------------------------------ MSE loss
__global__ void k_mse(const float* __restrict__ out, const float* __restrict__ target, const float* __restrict__ mask,
                      int C, int HW, double* __restrict__ loss, float* __restrict__ dout, const int* __restrict__ it_dev) {
  pdl_enter();
  const int n = C * HW;
  const float inv_n = 1.f / static_cast<float>(n);
  float acc = 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float m = mask != nullptr ? mask[i % HW] : 1.f;
    const float d = m * (out[i] - target[i]);
    acc = fmaf(d, d, acc);
    if (dout != nullptr) dout[i] = 2.f * m * d * inv_n;
  }
  __shared__ float red[32];
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    // each block's term rounded to a multiple of 2^-48: every partial sum below 32 is then exact in fp64, so the loss does
    // not depend on the order of the atomics; the rounding is <= 2^-49 per block, far below the fp32 error of `t` itself
    if (threadIdx.x == 0) {
      const double v = static_cast<double>(t) * static_cast<double>(inv_n);
      atomicAdd(loss + (it_dev != nullptr ? *it_dev : 0), ldexp(rint(ldexp(v, 48)), -48));
    }
  }
}
void launch_mse(const float* out, const float* target, const float* mask, int C, int HW, double* loss, float* dout,
                const int* it_dev, cudaStream_t s) {
  const long long n = static_cast<long long>(C) * HW;
  int blocks = static_cast<int>((n + 255) / 256);
  if (blocks > kNumSms * 4) blocks = kNumSms * 4;
  launch_k(k_mse, dim3(blocks), dim3(256), 0, s, 1, out, target, mask, C, HW, loss, dout, it_dev);
}

// ------------------------------------------------------------------------------------------------ Philox noise
__device__ __forceinline__ void philox_round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
  const uint32_t hi0 = __umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
  const uint32_t hi1 = __umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
  const uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
  c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
}
__global__ void k_noise(const float* __restrict__ z0, float* __restrict__ z, float sigma, uint64_t seed,
                        uint64_t offset, const int* __restrict__ it_dev, size_t n4) {
  pdl_enter();
  if (it_dev != nullptr) offset += static_cast<uint64_t>(*it_dev);
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    uint32_t c[4] = {static_cast<uint32_t>(i), static_cast<uint32_t>(i >> 32), static_cast<uint32_t>(offset),
                     static_cast<uint32_t>(offset >> 32)};
    uint32_t k0 = static_cast<uint32_t>(seed), k1 = static_cast<uint32_t>(seed >> 32);
#pragma unroll
    for (int r = 0; r < 10; ++r) {
      philox_round(c, k0, k1);
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    // Box-Muller on two pairs of uniforms in (0, 1]
    const float u0 = (static_cast<float>(c[0]) + 1.0f) * 2.3283064365386963e-10f;
    const float u1 = static_cast<float>(c[1]) * 2.3283064365386963e-10f;
    const float u2 = (static_cast<float>(c[2]) + 1.0f) * 2.3283064365386963e-10f;
    const float u3 = static_cast<float>(c[3]) * 2.3283064365386963e-10f;
    const float r0 = sqrtf(-2.f * __logf(u0)), r1 = sqrtf(-2.f * __logf(u2));
    float s0, c0, s1, c1;
    __sincosf(6.283185307179586f * u1, &s0, &c0);
    __sincosf(6.283185307179586f * u3, &s1, &c1);
    float4 zv = ld4(z0 + 4 * i);
    zv.x = fmaf(sigma, r0 * c0, zv.x);
    zv.y = fmaf(sigma, r0 * s0, zv.y);
    zv.z = fmaf(sigma, r1 * c1, zv.z);
    zv.w = fmaf(sigma, r1 * s1, zv.w);
    st4(z + 4 * i, zv);
  }
}
void launch_noise(const float* z0, float* z, float sigma, uint64_t seed, uint64_t offset, const int* it_dev, size_t n,
                  cudaStream_t s) {
  const size_t n4 = n / 4;
  int blocks = static_cast<int>((n4 + 255) / 256);
  if (blocks > kNumSms * 16) blocks = kNumSms * 16;
  launch_k(k_noise, dim3(blocks), dim3(256), 0, s, 1, z0, z, sigma, seed, offset, it_dev, n4);
}
// Fused runner input: z = z0 + sigma * N(0,1) written straight into the reflection-padded NHWC level-0 buffer (k_noise +
// k_input_pad in one pass: z is never materialised).  Same Philox stream as k_noise: counter = flat NCHW index / 4, the four
// outputs of a block go to four consecutive x of one (channel, row).  Block = one source row x 32 source columns; phase 1:
// thread (channel, group of 4 pixels) generates; phase 2: thread (channel, pixel) writes the interior position and every halo
// position that mirrors it (ReflectionPad2d(1): padded row 0 <- source row 1, row H+1 <- row H-2, same for columns).
// ZP (zero padding): the source pixels on the image border write zeros into the halo cells next to them instead.
template <bool ZP>
__global__ void __launch_bounds__(256) k_noise_pad(const float* __restrict__ z0, float sigma, uint64_t seed, uint64_t offset,
                                                   const int* __restrict__ it_dev, float* __restrict__ dst, int C, int H, int W,
                                                   int Cs, Twin t16) {
  pdl_enter();
  __shared__ float tile[32][33];   // [pixel][channel]
  if (it_dev != nullptr) offset += static_cast<uint64_t>(*it_dev);
  const int sy = blockIdx.y, x0 = blockIdx.x * 32, Wp = W + 2;
  const int gx = threadIdx.x & 7, cl = threadIdx.x >> 3;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int c0 = 0; c0 < C; c0 += 32) {
    const int c = c0 + cl, x = x0 + 4 * gx;
    float4 val = f4zero();
    if (c < Cs && x < W) {
      const size_t flat = (static_cast<size_t>(c) * H + sy) * W + x;
      const size_t i = flat >> 2;
      uint32_t ctr[4] = {static_cast<uint32_t>(i), static_cast<uint32_t>(i >> 32), static_cast<uint32_t>(offset),
                         static_cast<uint32_t>(offset >> 32)};
      uint32_t k0 = static_cast<uint32_t>(seed), k1 = static_cast<uint32_t>(seed >> 32);
#pragma unroll
      for (int r = 0; r < 10; ++r) {
        philox_round(ctr, k0, k1);
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
      }
      const float u0 = (static_cast<float>(ctr[0]) + 1.0f) * 2.3283064365386963e-10f;
      const float u1 = static_cast<float>(ctr[1]) * 2.3283064365386963e-10f;
      const float u2 = (static_cast<float>(ctr[2]) + 1.0f) * 2.3283064365386963e-10f;
      const float u3 = static_cast<float>(ctr[3]) * 2.3283064365386963e-10f;
      const float r0 = sqrtf(-2.f * __logf(u0)), r1 = sqrtf(-2.f * __logf(u2));
      float s0, cs0, s1, cs1;
      __sincosf(6.283185307179586f * u1, &s0, &cs0);
      __sincosf(6.283185307179586f * u3, &s1, &cs1);
      val = ld4(z0 + flat);
      val.x = fmaf(sigma, r0 * cs0, val.x);
      val.y = fmaf(sigma, r0 * s0, val.y);
      val.z = fmaf(sigma, r1 * cs1, val.z);
      val.w = fmaf(sigma, r1 * s1, val.w);
    }
    tile[4 * gx + 0][cl] = val.x;
    tile[4 * gx + 1][cl] = val.y;
    tile[4 * gx + 2][cl] = val.z;
    tile[4 * gx + 3][cl] = val.w;
    __syncthreads();
    if (c0 + tx < C) {
      int rows[3], nr = 0;
      rows[nr++] = sy + 1;
      if (sy == (ZP ? 0 : 1)) rows[nr++] = 0;
      if (sy == (ZP ? H - 1 : H - 2)) rows[nr++] = H + 1;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int pix = ty + 8 * k, sx = x0 + pix;
        if (sx >= W) continue;
        const float o = tile[pix][tx];
        int cols[3], nc = 0;
        cols[nc++] = sx + 1;
        if (sx == (ZP ? 0 : 1)) cols[nc++] = 0;
        if (sx == (ZP ? W - 1 : W - 2)) cols[nc++] = W + 1;
        for (int a = 0; a < nr; ++a)
          for (int b = 0; b < nc; ++b) {
            const float ob = ZP && (a > 0 || b > 0) ? 0.f : o;
            dst[(static_cast<size_t>(rows[a]) * Wp + cols[b]) * C + c0 + tx] = ob;
            if (t16.p != nullptr) t16.p[(static_cast<size_t>(rows[a]) * Wp + cols[b]) * t16.ld + c0 + tx] = bf16_bits(ob);
          }
      }
    }
    __syncthreads();
  }
}
void launch_noise_pad(const float* z0, float sigma, uint64_t seed, uint64_t offset, const int* it_dev, float* dst, int C, int H,
                      int W, int c_src, cudaStream_t s, Twin t16, int zero_pad) {
  dim3 grid((W + 31) / 32, H);
  launch_k(zero_pad ? k_noise_pad<true> : k_noise_pad<false>, dim3(grid), dim3(256), 0, s, 1, z0, sigma, seed, offset, it_dev, dst,
           C, H, W, c_src > 0 ? c_src : C, t16);
}
__global__ void k_advance(int* it) {
  pdl_enter(); it[0] += 1; it[1] += 1; }  // {global Adam step, iteration index of this call}
void launch_advance(int* it_dev, cudaStream_t s) { launch_k(k_advance, dim3(1), dim3(1), 0, s, 1, it_dev); }

// ------------------------------------------------------------------------------------------------ Adam
// Arithmetic order follows torch.optim.Adam (single-tensor path): m = lerp(m, g, 1-b1); v = v*b2 + (1-b2) g^2;
// p -= (lr/bc1) * m / (sqrt(v)/sqrt(bc2) + eps).  Bias corrections are evaluated in fp64 on the device so that the
// step number can come from a device counter (CUDA-graph replay).
// kTrack: the tracker's action (AdamTrack) selects where p comes from and whether it is saved; the untracked instantiation
// never reads `tr`.
static constexpr int kAdamChunk = 2048;
template <bool kTrack>
__global__ void k_adam(AdamTable t, double lr, double b1, double b2, double eps, int step, const int* __restrict__ it_dev,
                       AdamTrack tr) {
  pdl_enter();
  __shared__ float s_step_size, s_bc2_sqrt;
  __shared__ int s_action;
  if (threadIdx.x == 0) {
    const int st = step + (it_dev != nullptr ? *it_dev : 0);
    if (kTrack) s_action = tr.st->action;
    const double bc1 = 1.0 - pow(b1, static_cast<double>(st));
    const double bc2 = 1.0 - pow(b2, static_cast<double>(st));
    s_step_size = static_cast<float>(lr / bc1);
    s_bc2_sqrt = static_cast<float>(sqrt(bc2));
  }
  __syncthreads();
  const float step_size = s_step_size, bc2_sqrt = s_bc2_sqrt;
  const float w1 = static_cast<float>(1.0 - b1), fb2 = static_cast<float>(b2), w2 = static_cast<float>(1.0 - b2);
  const float feps = static_cast<float>(eps);
  const int ti = t.blk_tensor[blockIdx.x];
  const int start = t.blk_start[blockIdx.x];
  const int n = t.numel[ti];
  float* __restrict__ p = t.p[ti];
  const float* __restrict__ g = t.g[ti];
  float* __restrict__ m = t.m[ti];
  float* __restrict__ v = t.v[ti];
  const int end = min(start + kAdamChunk, n);
  if (!kTrack) {
    for (int i = start + threadIdx.x; i < end; i += blockDim.x) {
      const float gi = g[i];
      float mi = m[i];
      mi = mi + (gi - mi) * w1;
      const float vi = v[i] * fb2 + w2 * gi * gi;
      m[i] = mi;
      v[i] = vi;
      const float denom = sqrtf(vi) / bc2_sqrt + feps;
      p[i] = p[i] - step_size * (mi / denom);
    }
    return;
  }
  const int action = s_action;
  float* __restrict__ snap = tr.snapshot + tr.off[ti];
  const float* src = action == kTrackRestored ? snap : p;
  for (int i = start + threadIdx.x; i < end; i += blockDim.x) {
    const float gi = g[i];
    float mi = m[i];
    mi = mi + (gi - mi) * w1;
    const float vi = v[i] * fb2 + w2 * gi * gi;
    m[i] = mi;
    v[i] = vi;
    const float denom = sqrtf(vi) / bc2_sqrt + feps;
    const float pi = src[i];
    if (action == kTrackSaved) snap[i] = pi;
    p[i] = pi - step_size * (mi / denom);
  }
}
void launch_adam(AdamTable t, double lr, double b1, double b2, double eps, int step, const int* it_dev, cudaStream_t s) {
  launch_k(k_adam<false>, dim3(t.nblocks), dim3(256), 0, s, 1, t, lr, b1, b2, eps, step, it_dev, AdamTrack{});
}
void launch_adam_track(AdamTable t, double lr, double b1, double b2, double eps, int step, const int* it_dev, AdamTrack tr,
                       cudaStream_t s) {
  launch_k(k_adam<true>, dim3(t.nblocks), dim3(256), 0, s, 1, t, lr, b1, b2, eps, step, it_dev, tr);
}

// ------------------------------------------------------------------------------------------------ closure tracker
// denoising.ipynb c10:8-52 inside the captured step.  k_track_out: the EMA in torch's rounding (`out_avg * w + out * (1 - w)`
// on fp32 CUDA tensors: each scalar rounded to fp32, three separately rounded operations) and the two ground-truth MSEs
// with k_mse's reduction, so that they do not depend on block order either.
__global__ void k_track_out(const float* __restrict__ out, const float* __restrict__ gt, float* __restrict__ avg,
                            const TrackState* __restrict__ st, float w_avg, float w_out, int n, double* __restrict__ rec,
                            const int* __restrict__ it_dev) {
  pdl_enter();
  const bool first = st->has_avg == 0;
  const float inv_n = 1.f / static_cast<float>(n);
  float acc_out = 0.f, acc_avg = 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float o = out[i];
    const float a = first ? o : __fadd_rn(__fmul_rn(avg[i], w_avg), __fmul_rn(o, w_out));
    avg[i] = a;
    if (gt != nullptr) {
      const float g = gt[i];
      const float d0 = o - g, d1 = a - g;
      acc_out = fmaf(d0, d0, acc_out);
      acc_avg = fmaf(d1, d1, acc_avg);
    }
  }
  if (gt == nullptr) return;
  __shared__ float red[2][32];
  for (int o = 16; o > 0; o >>= 1) {
    acc_out += __shfl_xor_sync(0xffffffffu, acc_out, o);
    acc_avg += __shfl_xor_sync(0xffffffffu, acc_avg, o);
  }
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = acc_out; red[1][threadIdx.x >> 5] = acc_avg; }
  __syncthreads();
  if (threadIdx.x < 32) {
    float t0 = threadIdx.x < (blockDim.x >> 5) ? red[0][threadIdx.x] : 0.f;
    float t1 = threadIdx.x < (blockDim.x >> 5) ? red[1][threadIdx.x] : 0.f;
    for (int o = 16; o > 0; o >>= 1) {
      t0 += __shfl_xor_sync(0xffffffffu, t0, o);
      t1 += __shfl_xor_sync(0xffffffffu, t1, o);
    }
    if (threadIdx.x == 0) {   // as k_mse: each block's term rounded to a multiple of 2^-48
      double* r = rec + kTrackRecord * (it_dev != nullptr ? *it_dev : 0);
      atomicAdd(r + 2, ldexp(rint(ldexp(static_cast<double>(t0) * static_cast<double>(inv_n), 48)), -48));
      atomicAdd(r + 3, ldexp(rint(ldexp(static_cast<double>(t1) * static_cast<double>(inv_n), 48)), -48));
    }
  }
}
void launch_track_out(const float* out, const float* gt, float* out_avg, const TrackState* st, float w_avg, float w_out,
                      int n, double* rec, const int* it_dev, cudaStream_t s) {
  int blocks = (n + 255) / 256;   // launch_mse's grid: the same per-thread terms
  if (blocks > kNumSms * 4) blocks = kNumSms * 4;
  launch_k(k_track_out, dim3(blocks), dim3(256), 0, s, 1, out, gt, out_avg, st, w_avg, w_out, n, rec, it_dev);
}
// c10:41-52: PSNRs (skimage compare_psnr, data range 1) of the iteration's loss and sums, then the back-tracking rule.
// A restore leaves i and psnr_last alone; a drop with no snapshot yet saves.
__global__ void k_track_decide(const double* __restrict__ loss, double* __restrict__ rec, TrackState* __restrict__ st,
                               int show_every, double backtrack_db, int has_gt, const int* __restrict__ it_dev) {
  pdl_enter();
  if (threadIdx.x != 0) return;
  const int slot = it_dev != nullptr ? *it_dev : 0;
  double* r = rec + kTrackRecord * slot;
  const double l = loss[slot];
  const double psnr = -10.0 * log10(l);
  r[0] = l;
  r[1] = psnr;
  r[2] = has_gt ? -10.0 * log10(r[2]) : CUDART_NAN;
  r[3] = has_gt ? -10.0 * log10(r[3]) : CUDART_NAN;
  TrackState x = *st;
  r[4] = static_cast<double>(x.i);
  int action = kTrackNone;
  if (show_every > 0 && x.i % show_every != 0) {
    if (psnr - x.psnr_last < -backtrack_db && x.has_snapshot) {
      action = kTrackRestored;
      x.fallbacks += 1;
    } else {
      action = kTrackSaved;
      x.has_snapshot = 1;
      x.psnr_last = psnr;
      x.i += 1;
    }
  } else {
    x.i += 1;
  }
  x.action = action;
  x.has_avg = 1;
  *st = x;
  r[5] = static_cast<double>(action);
}
void launch_track_decide(const double* loss, double* rec, TrackState* st, int show_every, double backtrack_db, int has_gt,
                         const int* it_dev, cudaStream_t s) {
  launch_k(k_track_decide, dim3(1), dim3(32), 0, s, 1, loss, rec, st, show_every, backtrack_db, has_gt, it_dev);
}
int adam_chunk() { return kAdamChunk; }

}  // namespace dip
