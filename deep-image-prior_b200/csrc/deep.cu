// Persistent deep-level kernel: see deep.cuh.  This translation unit contains conv_tc.cu and kernels_mem.cu (their device
// code is inlined into the op interpreter below; their stand-alone kernels and launchers are compiled here too).
#include "conv_tc.cu"
#include "kernels_mem.cu"
#include "deep.cuh"

namespace dip {

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// Grid-wide barrier between two ops.  Every op's global writes (generic stores, fp64 atomics, TMA bulk stores) must be
// visible to every other CTA's reads of the next op (generic loads and TMA loads): proxy fence (generic <-> async) +
// release/acquire on the counter.  The counter only grows (epoch * gridDim.x): no reset race.  A watchdog traps instead of
// hanging the GPU if a CTA never arrives.
__device__ __forceinline__ void grid_sync(unsigned* bar, unsigned& epoch) {
  asm volatile("fence.proxy.async;" ::: "memory");
  __syncthreads();
  if (threadIdx.x == 0) {
    epoch += gridDim.x;
    __threadfence();
    atomicAdd(bar, 1u);
    unsigned long long spins = 0;
    while (ld_acquire_u32(bar) < epoch) {
      if (++spins > (1ull << 27)) __trap();
    }
    __threadfence();
  }
  __syncthreads();
  asm volatile("fence.proxy.async;" ::: "memory");
}

template <class T>
__device__ __forceinline__ void copy_to_smem(T* dst, const T* src) {
  static_assert(sizeof(T) % 4 == 0, "");
  for (int i = threadIdx.x; i < static_cast<int>(sizeof(T) / 4); i += blockDim.x)
    reinterpret_cast<int*>(dst)[i] = reinterpret_cast<const int*>(src)[i];
  __syncthreads();
}

__global__ void __launch_bounds__(256, 1) k_deep(const DeepOp* __restrict__ ops, int nops, unsigned* bar) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  __shared__ __align__(16) TcConvParams s_conv;
  __shared__ __align__(16) TcWgradParams s_wg;
  unsigned epoch = 0;
  for (int i = 0; i < nops; ++i) {
    const DeepOp* op = ops + i;
    const int type = op->type, VL = op->VL, PPB = op->PPB;
    switch (type) {
      case DO_CONV:
        copy_to_smem(&s_conv, &op->u.conv);
        tc_conv_body<true>(s_conv, &op->u.conv, smem_raw);
        break;
      case DO_WGRAD:
        copy_to_smem(&s_wg, &op->u.wg);
        tc_wgrad_body<true>(s_wg, &op->u.wg, smem_raw);
        break;
      case DO_SKINNY_FWD: {
        const DeepSkinnyFwd a = op->u.skf;
        d_skinny_fwd(a.x, a.ldx, a.x_rs, a.w, a.b, a.C, a.N, a.H, a.W, a.y, a.mode, a.stats, a.cw);
      } break;
      case DO_BN_ACT_WRITE: {
        const DeepBnActWrite a = op->u.bnw;
        d_bn_act_write(a.raw, a.ld_in, a.bn, a.H, a.W, a.dst, a.ld_out, a.pad, a.act, VL, PPB);
      } break;
      case DO_CAT_STATS: {
        const DeepCat a = op->u.cat;
        d_cat_stats(a.a, a.fwd, VL, PPB);
      } break;
      case DO_CAT_WRITE: {
        const DeepCat a = op->u.cat;
        d_cat_write(a.a, a.bn_cat, a.dst, VL, PPB);
      } break;
      case DO_BN_BWD_REDUCE: {
        const DeepBnBwd a = op->u.bnb;
        if (a.src.kind == 0) d_bn_bwd_reduce<0>(a.raw, a.ld_raw, a.bn, a.act, a.src, a.H, a.W, a.bwd, VL, PPB);
        else d_bn_bwd_reduce<1>(a.raw, a.ld_raw, a.bn, a.act, a.src, a.H, a.W, a.bwd, VL, PPB);
      } break;
      case DO_BN_BWD_APPLY: {
        const DeepBnBwd a = op->u.bnb;
        if (a.src.kind == 0) d_bn_bwd_apply<0>(a.raw, a.ld_raw, a.bn, a.act, a.src, a.H, a.W, a.bwd, a.draw, a.zs, a.dbias, VL, PPB);
        else d_bn_bwd_apply<1>(a.raw, a.ld_raw, a.bn, a.act, a.src, a.H, a.W, a.bwd, a.draw, a.zs, a.dbias, VL, PPB);
      } break;
      case DO_CAT_BWD_REDUCE: {
        const DeepCatBwd a = op->u.catb;
        d_cat_bwd_reduce(a.pcat, a.bn_cat, a.gp, a.ld, a.H, a.W, a.bwd, VL, PPB);
      } break;
      case DO_CAT_BWD_APPLY: {
        const DeepCatBwd a = op->u.catb;
        d_cat_bwd_apply(a.pcat, a.bn_cat, a.gp, a.ld, a.H, a.W, a.bwd, a.dcat, VL, PPB);
      } break;
      case DO_UPADJ: {
        const DeepUpadj a = op->u.up;
        d_upadj(a.D, a.ld, a.coff, a.h, a.w, a.C, a.bilinear, a.dst, VL, PPB);
      } break;
      case DO_SKINNY_BWD: {
        const DeepSkinnyBwd a = op->u.skb;
        d_skinny_bwd(a.x, a.ldx, a.x_rs, a.w, a.C, a.N, a.H, a.W, a.dy, a.out_nchw, a.mode, a.dx, a.dw, a.db, VL, PPB, a.cw);
      } break;
      default: break;
    }
    if (op->sync) grid_sync(bar, epoch); else __syncthreads();
  }
}

static size_t g_deep_dyn = 0;
size_t deep_dyn_smem() {
  if (g_deep_dyn == 0) {
    cudaFuncAttributes at{};
    if (cudaFuncGetAttributes(&at, k_deep) != cudaSuccess) return 0;
    const size_t lim = 232448;   // 227 KB per CTA
    g_deep_dyn = ((lim - at.sharedSizeBytes) / 1024) * 1024;
  }
  return g_deep_dyn;
}
cudaError_t deep_kernels_init() {
  const size_t dyn = deep_dyn_smem();
  if (dyn == 0) return cudaErrorUnknown;
  return cudaFuncSetAttribute(k_deep, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(dyn));
}
cudaError_t launch_deep(const DeepOp* ops, int nops, unsigned* bar, int grid, cudaStream_t s) {
  cudaError_t e = cudaMemsetAsync(bar, 0, sizeof(unsigned), s);
  if (e != cudaSuccess) return e;
  return launch_k(k_deep, dim3(grid), dim3(256), deep_dyn_smem(), s, 1, ops, nops, bar);
}

}  // namespace dip
