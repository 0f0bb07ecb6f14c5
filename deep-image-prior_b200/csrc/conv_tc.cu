// wgmma / TMA implicit-GEMM convolution kernels for sm_90a (hand-written, no CUTLASS).
//
// Replaces what torch.nn.Conv2d forward/backward computes for the skip network
// (reference call site: models/common.py:120 via models/skip.py:58,64,68,83,89; backward = autograd of same).
//
//   tc_conv_kernel  : fprop and dgrad.  Persistent, warp-specialised, 256 threads:
//                       warp 0     TMA producer (im2col folded into the tensor-map coordinates: one 5-D box per tap)
//                       warp 3     loads the bias
//                       warps 4-7  one warpgroup: wgmma on the 128-pixel tile (two m64 halves, fp32 accumulators in
//                                  registers), then the epilogue: +bias -> swizzled smem -> per-channel BN statistics -> TMA store
//   tc_wgrad_kernel : weight gradient, split-K over work items (tap, pixel range), one partial slice per item.  dY and X arrive
//                     pixel-major from NHWC activations.  tf32: warps 4-7 read dY straight into wgmma A registers; wgmma reads
//                     a shared-memory tf32 B K-major only, so warps 1-3 transpose X into a double-buffered K-major tile while
//                     the previous block multiplies.  bf16: the warpgroup transposes both operands, then multiplies.
//   Both are templated on the operand type: tf32 on fp32 tensors (tc_conv_kernel / tc_wgrad_kernel) and bf16 on bf16 twins
//   (tc_conv_kernel_bf16 / tc_wgrad_kernel_bf16, precision mode bf16); accumulators and outputs are fp32 in both.
#include "conv_tc.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"
#include "kernels.cuh"

namespace dip {

static constexpr int kTileM = 128;            // output pixels per tile (two wgmma m64 halves)
static constexpr int kABytes = kTileM * 128;  // one A stage: 128 rows x 128 bytes
static constexpr int kChunkBytes = kTileM * 128;
static constexpr int kNumThreads = 256;
static constexpr int kAccStride = kAccS;  // fp64 accumulators: kAccR replicas x one 128-byte line each (kernels.cuh)

struct SmemCtl {
  uint64_t full[8];
  uint64_t empty[8];
  float bias[160];
};

__host__ __device__ constexpr int round32(int n) { return (n + 31) & ~31; }
__host__ __device__ constexpr int round1024(int n) { return (n + 1023) & ~1023; }

// ------------------------------------------------------------------------------------------------ fprop / dgrad
template <int NT>
__device__ __forceinline__ void tc_conv_epilogue(const TcConvParams& p, SmemCtl* ctl, uint8_t* staging,
                                                 float (&acc)[2][NT / 2], int x0, int y0, int opx, int opy, int n_off,
                                                 double& stat_s1, double& stat_s2, bool col_halves = false);
__device__ __forceinline__ void tc_conv_stats_flush(const TcConvParams& p, int n_off, double stat_s1, double stat_s2);

// Consumer warpgroup (threads 128..255) of the conv kernel, NT = wgmma N (n_mma rounded up to 32).
template <bool BF16, int NT>
__device__ __forceinline__ void tc_conv_consumer(const TcConvParams& p, SmemCtl* ctl,
                                                 uint8_t* stage_base, int stage_bytes, uint8_t* staging, int n_iters,
                                                 int tile0, int tile_stride, int num_tiles, int tiles_pp, int n_off) {
  const int lane = threadIdx.x & 31;
  float acc[2][NT / 2];
  int stage = 0;
  uint32_t phase = 0;
  double stat_s1 = 0.0, stat_s2 = 0.0;
  const uint32_t base_lo = desc_lo(smem_u32(stage_base));
  const uint32_t stage_step = static_cast<uint32_t>(stage_bytes) >> 4;
  constexpr uint32_t kBOff = static_cast<uint32_t>(kABytes) >> 4;
  constexpr uint32_t kHalfOff = (64u * 128u) >> 4;   // second m64 half of the A tile
  for (int it = 0; it < n_iters; ++it) {
    const int tile = tile0 + it * tile_stride;
    int tx = tile % p.tiles_x, ty = tile / p.tiles_x;
    int opx = 0, opy = 0;
    int kb_per_tile = p.kh * p.kw * p.kblocks;
    if (p.nphase > 0) {
      if (tile >= num_tiles) break;
      const int t = tile % tiles_pp;
      tx = t % p.tiles_x; ty = t / p.tiles_x;
      const TcConvParams::Phase& q = p.phs[tile / tiles_pp];
      opx = q.opx; opy = q.opy;
      kb_per_tile = q.kh * q.kw * p.kblocks;
    }
    const int x0 = tx * p.bw, y0 = ty * p.bh;
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
    int prev = -1;
    for (int kbt = 0; kbt < kb_per_tile; ++kbt) {
      mbar_wait(&ctl->full[stage], phase);
      const uint32_t a_lo = base_lo + stage * stage_step;
      const uint32_t b_lo = a_lo + kBOff;
      // all four K steps of every block: channels past C are zero in both operands (TMA zero-fills the activation past
      // its channel extent, the packed weights are zero there), so a partial last block needs no shorter issue sequence
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {   // K-major SW128: advancing K by 8 fp32 / 16 bf16 = +32 B inside the swizzle atom
        wgmma_ss<NT, BF16>(acc[0], desc_of(a_lo + 2 * k), desc_of(b_lo + 2 * k));
        wgmma_ss<NT, BF16>(acc[1], desc_of(a_lo + kHalfOff + 2 * k), desc_of(b_lo + 2 * k));
      }
      wgmma_commit();
      if (prev >= 0) {   // the previous stage's wgmmas have read their operands -> hand it back to the producer
        wgmma_wait<1>();
        if (lane == 0) mbar_arrive(&ctl->empty[prev]);
      }
      prev = stage;
      if (++stage == p.stages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    if (prev >= 0 && lane == 0) mbar_arrive(&ctl->empty[prev]);
    tc_conv_epilogue<NT>(p, ctl, staging, acc, x0, y0, opx, opy, n_off, stat_s1, stat_s2);
  }
  tc_conv_stats_flush(p, n_off, stat_s1, stat_s2);
}

// Epilogue of one tile (consumer warpgroup): + bias -> swizzled staging -> TMA store, and the tile's per-channel
// statistics added to the running totals s1 / s2.
template <int NT>
__device__ __forceinline__ void tc_conv_epilogue(const TcConvParams& p, SmemCtl* ctl, uint8_t* staging,
                                                 float (&acc)[2][NT / 2], int x0, int y0, int opx, int opy, int n_off,
                                                 double& stat_s1, double& stat_s2, bool col_halves) {
  const int et = threadIdx.x - 128;    // 0..127
  const int w = et >> 5, lane = et & 31;
  const int bw_shift = 31 - __clz(p.bw);  // tile widths are powers of two
  {
    // staging buffer must be free (previous tile's TMA store has finished reading it)
    if (et == 0) tma_store_wait_read0();
    named_bar_sync(1, 128);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int j = 0; j < NT / 8; ++j) {
        const int col = 8 * j + 2 * (lane & 3);
        const int chunk = col >> 5;
        if (chunk < p.n_chunks) {
          const int q = (col & 31) >> 2, e = col & 3;
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            // accumulator row -> staging row (pixel py * bw + px): the m64 halves are the tile's two row halves, or, for the
            // 16-wide tiles of the patch path (col_halves), its two 8-pixel column halves
            const int r64 = 16 * w + (lane >> 2) + 8 * rr;
            const int row = col_halves ? ((r64 >> 3) << 4) + 8 * h + (r64 & 7) : 64 * h + r64;
            float2 o;
            o.x = acc[h][4 * j + 2 * rr] + ctl->bias[col];
            o.y = acc[h][4 * j + 2 * rr + 1] + ctl->bias[col + 1];
            *reinterpret_cast<float2*>(staging + chunk * kChunkBytes + row * 128 + ((q ^ (row & 7)) << 4) + e * 4) = o;
          }
        }
      }
    }
    fence_proxy_async_smem();
    named_bar_sync(1, 128);
    if (et == 0) {
      if (p.nphase > 0)
        for (int j = 0; j < p.n_chunks; ++j) tma_store_5d(&p.tmD, staging + j * kChunkBytes, n_off + j * 32, opx, x0, opy, y0);
      else
        for (int j = 0; j < p.n_chunks; ++j) tma_store_3d(&p.tmD, staging + j * kChunkBytes, n_off + j * 32, x0, y0);
      tma_store_commit();
    }
    if (p.stats != nullptr && et < p.n_mma) {
      // per-channel sum / sum-of-squares of this tile (feeds the following BatchNorm): thread = channel et, running
      // totals stay in registers across all tiles of this persistent CTA (one fp64 atomic pair per thread at the end)
      const int c = et;
      const int j = c >> 5, q = (c & 31) >> 2, e = c & 3;
      const uint8_t* cb = staging + j * kChunkBytes + e * 4;
      float a0 = 0.f, a1 = 0.f, b0 = 0.f, b1 = 0.f;
      if (x0 + p.bw <= p.out_w && y0 + p.bh <= p.out_h) {
#pragma unroll 8
        for (int m = 0; m < kTileM; m += 2) {
          const float x = *reinterpret_cast<const float*>(cb + m * 128 + ((q ^ (m & 7)) << 4));
          const float y = *reinterpret_cast<const float*>(cb + (m + 1) * 128 + ((q ^ ((m + 1) & 7)) << 4));
          a0 += x; b0 = fmaf(x, x, b0);
          a1 += y; b1 = fmaf(y, y, b1);
        }
      } else {
        for (int m = 0; m < kTileM; ++m) {
          const int py = m >> bw_shift, px = m & (p.bw - 1);
          if (x0 + px < p.out_w && y0 + py < p.out_h) {
            const float x = *reinterpret_cast<const float*>(cb + m * 128 + ((q ^ (m & 7)) << 4));
            a0 += x; b0 = fmaf(x, x, b0);
          }
        }
      }
      stat_s1 += static_cast<double>(a0 + a1);
      stat_s2 += static_cast<double>(b0 + b1);
    }
  }
}

// End of the consumer warpgroup's work: one fp64 atomic pair per channel, then wait for the last TMA store.
__device__ __forceinline__ void tc_conv_stats_flush(const TcConvParams& p, int n_off, double stat_s1, double stat_s2) {
  const int et = threadIdx.x - 128;
  if (p.stats != nullptr && et < p.n_mma && n_off + et < p.stats_ld) {
    const int rep = (blockIdx.x % kAccR) * kAccLine;
    atomicAdd(&p.stats[(n_off + et) * kAccStride + rep], stat_s1);
    atomicAdd(&p.stats[(p.stats_ld + n_off + et) * kAccStride + rep], stat_s2);
  }
  if (et == 0) tma_store_wait_all0();
}

// Body of the conv kernel.  BF16 = true: operands are bf16 (K = 16 per wgmma).  The BYTE geometry is unchanged -- an operand
// row is still 128 bytes, now 64 channels, and one wgmma still advances 32 bytes along K -- so a "k block" is 64 channels,
// p.kblocks counts those, and only the channel coordinate of the TMA boxes and the instruction type differ.
template <bool BF16>
__device__ __forceinline__ void tc_conv_body(const TcConvParams& p, uint8_t* smem_raw) {
  constexpr int KE = BF16 ? 64 : 32;   // channels per 128-byte operand row
  // 1024-byte alignment is required by the 128B swizzle atoms.
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int nt = round32(p.n_mma);
  const int b_bytes = p.n_mma * 128;                       // bytes TMA writes per B tile
  const int stage_bytes = kABytes + round1024(nt * 128);   // [A tile 16 KB][B tile, room for nt rows]
  // layout: [stages | epilogue staging | control], stages and staging 1024-byte aligned (swizzle atoms)
  uint8_t* stage_base = smem;
  uint8_t* staging = stage_base + p.stages * stage_bytes;
  SmemCtl* ctl = reinterpret_cast<SmemCtl*>(staging + p.n_chunks * kChunkBytes);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int tiles_pp = p.tiles_x * p.tiles_y;                     // tiles per sub-pixel phase (nphase > 0)
  const int num_tiles = p.nphase > 0 ? tiles_pp * p.nphase : tiles_pp;
  // N split (small levels, fewer tiles than SMs): n_split CTAs share a pixel tile, each computes n_mma = N / n_split
  // output channels -> each CTA ingests 1/n_split of the weights and the tile's work spreads over more SMs.
  // CTA = (tile slot, n_part); n_split == 1: slots == gridDim.x.
  const int n_split = p.n_split < 1 ? 1 : p.n_split;
  const int n_part = blockIdx.x % n_split;
  const int n_off = n_part * p.n_mma;             // first output channel of this CTA
  const int n_total = p.n_mma * n_split;          // rows per tap of the packed weights
  const int tile_stride = static_cast<int>(gridDim.x) / n_split;
  const int n_iters = (num_tiles + tile_stride - 1) / tile_stride;
  const int tile0 = blockIdx.x / n_split;         // first tile; stride tile_stride

  pdl_trigger();
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&p.tmA);
    tma_prefetch_desc(&p.tmB);
    tma_prefetch_desc(&p.tmD);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < p.stages; ++i) {
      mbar_init(&ctl->full[i], 1);
      mbar_init(&ctl->empty[i], 4);   // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  pdl_wait();  // everything above is independent of the previous kernel's results
  if (warp == 3) {
    for (int i = lane; i < 160; i += 32)
      ctl->bias[i] = (p.bias != nullptr && i < p.n_mma && (p.n_valid == 0 || n_off + i < p.n_valid)) ? p.bias[n_off + i] : 0.f;
  }
  __syncthreads();

  if (warp == 0) {
    // ===================================================================== TMA producer
    // The whole warp walks the loop (warp-uniform control flow); one elected lane issues the TMA instructions.
    int stage = 0;
    uint32_t phase = 0;
    for (int it = 0; it < n_iters; ++it) {
      const int tile = tile0 + it * tile_stride;
      // one phase (kh x kw taps at offx / offy) or the phase this work item belongs to
      int kh = p.kh, kw = p.kw, offx = p.offx, offy = p.offy, tap0 = 0;
      int x0 = (tile % p.tiles_x) * p.bw, y0 = (tile / p.tiles_x) * p.bh;
      if (p.nphase > 0) {
        if (tile >= num_tiles) break;
        const TcConvParams::Phase& q = p.phs[tile / tiles_pp];
        const int t = tile % tiles_pp;
        kh = q.kh; kw = q.kw; offx = q.offx; offy = q.offy; tap0 = q.tap0;
        x0 = (t % p.tiles_x) * p.bw; y0 = (t / p.tiles_x) * p.bh;
      }
      for (int r = 0; r < kh; ++r) {
        for (int s = 0; s < kw; ++s) {
          const int ix = offx + s, iy = offy + r;  // tap offset in input coordinates
          int cpx, cx, cpy, cy;
          if (p.stride == 1) {
            cpx = 0; cx = x0 + ix; cpy = 0; cy = y0 + iy;
          } else {
            // input coordinate = 2*out + i  ->  (parity, half) = (i & 1, out + (i >> 1)); offsets are >= 0 here
            cpx = ix & 1; cx = x0 + (ix >> 1); cpy = iy & 1; cy = y0 + (iy >> 1);
          }
          const int tap = tap0 + r * kw + s;
          for (int kb = 0; kb < p.kblocks; ++kb) {
            mbar_wait(&ctl->empty[stage], phase ^ 1);
            uint8_t* sa = stage_base + stage * stage_bytes;
            if (elect_one()) {
              mbar_expect_tx(&ctl->full[stage], kABytes + b_bytes);
              tma_load_5d(sa, &p.tmA, &ctl->full[stage], kb * KE, cpx, cx, cpy, cy);
              tma_load_2d(sa + kABytes, &p.tmB, &ctl->full[stage], kb * KE, tap * n_total + n_off);
            }
            __syncwarp();
            if (++stage == p.stages) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else if (warp >= 4) {
    // ===================================================================== wgmma + epilogue (one warpgroup)
    switch (nt) {
      case 32: tc_conv_consumer<BF16, 32>(p, ctl, stage_base, stage_bytes, staging, n_iters, tile0, tile_stride, num_tiles, tiles_pp, n_off); break;
      case 64: tc_conv_consumer<BF16, 64>(p, ctl, stage_base, stage_bytes, staging, n_iters, tile0, tile_stride, num_tiles, tiles_pp, n_off); break;
      case 96: tc_conv_consumer<BF16, 96>(p, ctl, stage_base, stage_bytes, staging, n_iters, tile0, tile_stride, num_tiles, tiles_pp, n_off); break;
      case 128: tc_conv_consumer<BF16, 128>(p, ctl, stage_base, stage_bytes, staging, n_iters, tile0, tile_stride, num_tiles, tiles_pp, n_off); break;
      default: tc_conv_consumer<BF16, 160>(p, ctl, stage_base, stage_bytes, staging, n_iters, tile0, tile_stride, num_tiles, tiles_pp, n_off); break;
    }
  }
  __syncthreads();
}
__global__ void __launch_bounds__(kNumThreads, 1) tc_conv_kernel(const __grid_constant__ TcConvParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  tc_conv_body<false>(p, smem_raw);
}
__global__ void __launch_bounds__(kNumThreads, 1) tc_conv_kernel_bf16(const __grid_constant__ TcConvParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  tc_conv_body<true>(p, smem_raw);
}

// ------------------------------------------------------------------------------------------------ stride-1 3x3 patch path
// tc_conv_patch_kernel: tc_conv_kernel for stride-1 3x3 convolutions (fprop and the stride-1 dgrad) on tiles 8 or 16
// pixels wide, with the same tiles, warp roles, weight stages, wgmma sequence and epilogue -- only the activation operand
// arrives differently.  Instead of one shifted 128-pixel tile per tap and K block, the producer loads, per tile and K
// block, the (bh + 2) x (bw + 2) = 180 pixel input patch ONCE, and the nine taps read it at nine offsets.  All K blocks of
// a tile stay resident (one patch slot per K block, each with its own pfull / pempty barrier), so the wgmmas run in
// exactly tc_conv_kernel's order -- taps outer, K blocks inner -- and every accumulator receives the same sums in the same
// order: the results are those of tc_conv_kernel, bit for bit.
// Layout: TMA writes a patch unswizzled as [16-byte channel group][patch row][patch col][16 B], so a wgmma core matrix
// (8 rows x 16 B) is 8 consecutive pixels of one patch row, contiguous at any pixel offset.  The two m64 halves of the
// tile are eight 8-pixel segments at a constant stride of one patch row: the eight rows 8h .. 8h + 7 of an 8 x 16 tile,
// or the eight rows of column half h (pixels 8h .. 8h + 7) of a 16 x 8 tile.  The A descriptor of tap (r, s), half h and
// K step k is then
//   start = patch + (r * PW + s + half_off(h)) * 16 B + k * 2 * plane,   SBO = PW * 16 B (one patch row),   LBO = plane
// (PW = bw + 2, half_off = 8 PW h for bw = 8 and 8 h for bw = 16, plane = one channel group of the patch, kPatchPlane); the
// epilogue maps accumulator rows back to staging rows py * bw + px.  The weights keep their 128-byte-swizzled stages.
// L2 -> SM bytes per tile and K block: 22.5 KB of activation + 9 weight tiles, instead of 9 x (16 KB + weight tile).
// wgmma N of the patch path: n_mma rounded up to 32, except 144 (the input gradient of the 128 + 4 channel concat convs,
// 144 = 132 rounded up to 16), which would otherwise give 16 zero columns and 2 KB of every weight stage to rounding
__host__ __device__ constexpr int patch_nt(int n_mma) { return n_mma == 144 ? 144 : round32(n_mma); }
struct PatchCtl {
  uint64_t pfull[kPatchMaxKb];
  uint64_t pempty[kPatchMaxKb];
};

// Trip counts of one CTA, shared by the producer and the consumer (both walk tiles, then the 9 taps, then K blocks).
struct PatchWork {
  int tile0, tile_stride, n_iters, n_off, n_total;
};
__device__ __forceinline__ PatchWork patch_work(const TcConvParams& p) {
  const int n_split = p.n_split < 1 ? 1 : p.n_split;
  PatchWork w;
  const int num_tiles = p.tiles_x * p.tiles_y;
  w.tile_stride = static_cast<int>(gridDim.x) / n_split;
  w.tile0 = blockIdx.x / n_split;
  w.n_iters = (num_tiles - w.tile0 + w.tile_stride - 1) / w.tile_stride;   // tiles tile0, tile0 + stride, ... < num_tiles
  w.n_off = static_cast<int>(blockIdx.x % n_split) * p.n_mma;
  w.n_total = p.n_mma * n_split;
  return w;
}
static constexpr int kPatchTaps = 9;

template <bool BF16, int NT>
__device__ __forceinline__ void tc_conv_patch_consumer(const TcConvParams& p, SmemCtl* ctl, PatchCtl* pc,
                                                       uint8_t* patch_base, uint8_t* b_base, int b_stage_bytes,
                                                       uint8_t* staging, const PatchWork& wk) {
  const int lane = threadIdx.x & 31;
  float acc[2][NT / 2];
  int stage = 0;
  uint32_t phase = 0, pphase = 0;
  double stat_s1 = 0.0, stat_s2 = 0.0;
  const uint32_t patch16 = smem_u32(patch_base) >> 4;
  const uint32_t b_lo0 = desc_lo(smem_u32(b_base));
  const uint32_t b_step = static_cast<uint32_t>(b_stage_bytes) >> 4;
  constexpr uint32_t kPlane16 = kPatchPlane >> 4, kSlot16 = kPatchBytes >> 4;
  const uint32_t row16 = p.bw + 2;                              // one patch row, in 16-byte units
  const uint32_t half16 = p.bw == 8 ? 8 * row16 : 8;            // second m64 half: 8 rows down, or 8 pixels right
  for (int it = 0; it < wk.n_iters; ++it) {
    const int tile = wk.tile0 + it * wk.tile_stride;
    const int x0 = (tile % p.tiles_x) * p.bw, y0 = (tile / p.tiles_x) * p.bh;
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
    int prev = -1;         // B stage read by the previous wgmma group
    int prev_patch = -1;   // patch slot read by the previous group if it was that slot's last (tap 8)
#pragma unroll 1
    for (int tap = 0; tap < kPatchTaps; ++tap) {
      const int r = tap / 3, s = tap - 3 * (tap / 3);
#pragma unroll 1
      for (int kb = 0; kb < p.kblocks; ++kb) {
        if (tap == 0) mbar_wait(&pc->pfull[kb], pphase);
        mbar_wait(&ctl->full[stage], phase);
        const uint32_t b_lo = b_lo0 + stage * b_step;
        const uint32_t a16 = patch16 + kb * kSlot16 + r * row16 + s;
        // all four K steps of every block, as in tc_conv_consumer (channels past the K extent are zero in both operands)
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          wgmma_ss<NT, BF16>(acc[0], desc_noswz(a16 + 2 * k * kPlane16, kPlane16, row16), desc_of(b_lo + 2 * k));
          wgmma_ss<NT, BF16>(acc[1], desc_noswz(a16 + half16 + 2 * k * kPlane16, kPlane16, row16), desc_of(b_lo + 2 * k));
        }
        wgmma_commit();
        if (prev >= 0) {   // the previous group's wgmmas have read their operands -> hand them back to the producer
          wgmma_wait<1>();
          if (lane == 0) {
            mbar_arrive(&ctl->empty[prev]);
            if (prev_patch >= 0) mbar_arrive(&pc->pempty[prev_patch]);
          }
        }
        prev = stage;
        prev_patch = tap == kPatchTaps - 1 ? kb : -1;
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
      }
    }
    pphase ^= 1;
    wgmma_wait<0>();
    if (prev >= 0 && lane == 0) {
      mbar_arrive(&ctl->empty[prev]);
      if (prev_patch >= 0) mbar_arrive(&pc->pempty[prev_patch]);
    }
    tc_conv_epilogue<NT>(p, ctl, staging, acc, x0, y0, 0, 0, wk.n_off, stat_s1, stat_s2, p.bw == 16);
  }
  tc_conv_stats_flush(p, wk.n_off, stat_s1, stat_s2);
}

template <bool BF16>
__device__ __forceinline__ void tc_conv_patch_body(const TcConvParams& p, uint8_t* smem_raw) {
  constexpr int KE = BF16 ? 64 : 32;   // channels per 128-byte operand row
  constexpr int KG = BF16 ? 8 : 4;     // channels per 16-byte group
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int nt = patch_nt(p.n_mma);
  const int b_bytes = p.n_mma * 128;
  const int b_stage_bytes = round1024(nt * 128);
  // layout: [B stages | epilogue staging | one patch per K block | control]; stages and staging 1024-byte aligned (swizzle
  // atoms), patches 128-byte aligned (kPatchBytes is a multiple of 128)
  uint8_t* b_base = smem;
  uint8_t* staging = b_base + p.stages * b_stage_bytes;
  uint8_t* patch_base = staging + p.n_chunks * kChunkBytes;
  SmemCtl* ctl = reinterpret_cast<SmemCtl*>(patch_base + p.kblocks * kPatchBytes);
  PatchCtl* pc = reinterpret_cast<PatchCtl*>(ctl + 1);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const PatchWork wk = patch_work(p);

  pdl_trigger();
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&p.tmA);
    tma_prefetch_desc(&p.tmB);
    tma_prefetch_desc(&p.tmD);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < p.stages; ++i) {
      mbar_init(&ctl->full[i], 1);
      mbar_init(&ctl->empty[i], 4);   // one arrival per consumer warp
    }
    for (int i = 0; i < p.kblocks; ++i) {
      mbar_init(&pc->pfull[i], 1);
      mbar_init(&pc->pempty[i], 4);
    }
    fence_mbar_init();
  }
  pdl_wait();
  if (warp == 3) {
    for (int i = lane; i < 160; i += 32)
      ctl->bias[i] = (p.bias != nullptr && i < p.n_mma && (p.n_valid == 0 || wk.n_off + i < p.n_valid)) ? p.bias[wk.n_off + i] : 0.f;
  }
  __syncthreads();

  if (warp == 0) {
    // ===================================================================== TMA producer
    // The whole warp walks the loop (warp-uniform control flow); one elected lane issues the TMA instructions.
    int stage = 0;
    uint32_t phase = 0, pphase = 0;
    for (int it = 0; it < wk.n_iters; ++it) {
      const int tile = wk.tile0 + it * wk.tile_stride;
      const int x0 = (tile % p.tiles_x) * p.bw, y0 = (tile / p.tiles_x) * p.bh;
      for (int tap = 0; tap < kPatchTaps; ++tap) {
        for (int kb = 0; kb < p.kblocks; ++kb) {
          if (tap == 0) {
            // patch slot kb is free once the previous tile's last tap has read it
            mbar_wait(&pc->pempty[kb], pphase ^ 1);
            if (elect_one()) {
              // out-of-range pixels (image border, dgrad's negative offsets, ragged tiles) and channels past C arrive as zeros
              mbar_expect_tx(&pc->pfull[kb], kPatchBytes);
              tma_load_4d(patch_base + kb * kPatchBytes, &p.tmA, &pc->pfull[kb], 0, x0 + p.offx, y0 + p.offy, kb * (KE / KG));
            }
            __syncwarp();
          }
          mbar_wait(&ctl->empty[stage], phase ^ 1);
          if (elect_one()) {
            mbar_expect_tx(&ctl->full[stage], b_bytes);
            tma_load_2d(b_base + stage * b_stage_bytes, &p.tmB, &ctl->full[stage], kb * KE, tap * wk.n_total + wk.n_off);
          }
          __syncwarp();
          if (++stage == p.stages) { stage = 0; phase ^= 1; }
        }
      }
      pphase ^= 1;
    }
  } else if (warp >= 4) {
    // ===================================================================== wgmma + epilogue (one warpgroup)
    switch (nt) {
      case 32: tc_conv_patch_consumer<BF16, 32>(p, ctl, pc, patch_base, b_base, b_stage_bytes, staging, wk); break;
      case 64: tc_conv_patch_consumer<BF16, 64>(p, ctl, pc, patch_base, b_base, b_stage_bytes, staging, wk); break;
      case 96: tc_conv_patch_consumer<BF16, 96>(p, ctl, pc, patch_base, b_base, b_stage_bytes, staging, wk); break;
      case 128: tc_conv_patch_consumer<BF16, 128>(p, ctl, pc, patch_base, b_base, b_stage_bytes, staging, wk); break;
      case 144: tc_conv_patch_consumer<BF16, 144>(p, ctl, pc, patch_base, b_base, b_stage_bytes, staging, wk); break;
      default: tc_conv_patch_consumer<BF16, 160>(p, ctl, pc, patch_base, b_base, b_stage_bytes, staging, wk); break;
    }
  }
  __syncthreads();
}
__global__ void __launch_bounds__(kNumThreads, 1) tc_conv_patch_kernel(const __grid_constant__ TcConvParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  tc_conv_patch_body<false>(p, smem_raw);
}
__global__ void __launch_bounds__(kNumThreads, 1) tc_conv_patch_kernel_bf16(const __grid_constant__ TcConvParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  tc_conv_patch_body<true>(p, smem_raw);
}

// ------------------------------------------------------------------------------------------------ wgrad
struct SmemCtlW {
  uint64_t full[8];
  uint64_t empty[8];
  uint64_t bt_full[2];    // tf32: the transposer warps have written Bt buffer i
  uint64_t bt_empty[2];   // tf32: the wgmmas that read Bt buffer i have completed
};

// Shared-memory bytes of one transposed operand buffer: [At, bf16 only: 128 rows][Bt: n_cols rows], 128 bytes a row.
__host__ __device__ constexpr int wgrad_tbuf_bytes(bool bf16, int n_cols) {
  return (bf16 ? kTileM * 128 : 0) + round1024(n_cols * 128);
}

// The tf32 weight gradient, per 32-pixel block of a work item: D[n][c] += dY[px][n]^T * X[px][c] over the block's pixels.
// A = dY^T (M = the 128 output channels) is read straight from the pixel-major TMA stage into registers (register-A wgmma);
// B = X^T must be K-major in shared memory, so warps 1-3 transpose the X stage into a double-buffered Bt tile while warps
// 4-7 run the wgmmas of the previous block.
//
// K order: inside every k8 step (pixels 8kk .. 8kk+7) K position j holds pixel 8kk + 2j for j < 4 and 8kk + 2(j-4) + 1 for
// j >= 4 -- even pixels first.  A and B use the same order, so the product is unchanged (the accumulation order inside one
// wgmma is the hardware's); it is the order that makes both the A-fragment loads and the transpose conflict-free (below).
//
// Stage layout (both operands): 128-byte rows of 32 fp32 channels, one row per pixel, chunks of 32 rows (4096 B) per 32
// channels, 16-byte group q of row px stored at slot q ^ (px & 7) (the TMA 128-byte swizzle).

// Warps 1-3 (96 threads): X stage -> Bt[NT rows = channels][32 pixels in the K order above], K-major SW128.
// A unit is 4 channels (group c4) x 4 pixels (8kk + e + 2i, i = 0..3): four LDS.128 (one per pixel, 4 channels each), a 4x4
// register transpose, four STS.128 (one per channel, 4 pixels each) into 16-byte group 2kk + e of the channel's Bt row.
// Bank argument: the 8 lanes that share a 128-bit shared-memory wavefront are b = lane & 7, with e = b0, c4 bits 1,2 = b1,b2,
// and kk = (b1 ^ o0) | (b2 ^ o1) << 1, c4 bit 0 = o2 for the lane-independent unit index o.  An LDS.128 of pixel 8kk + e + 2i
// hits slot (c4 & 7) ^ (e + 2i), whose bits are (o2 ^ b0, b1 ^ i0, b2 ^ i1): 8 distinct slots over b.  An STS.128 of channel
// 4 c4 + r hits slot (2kk + e) ^ (4 (c4 & 1) + r), bits (b0 ^ r0, b1 ^ o0 ^ r1, b2 ^ o1 ^ o2): 8 distinct slots over b.
// Both are conflict-free.  Units cover (c4 < NT / 4) x (kk < 4) x (e < 2) exactly once.
template <int NT>
__device__ __forceinline__ void tc_wgrad_transposer(const TcWgradParams& p, SmemCtlW* ctl, uint32_t stage_base, int stage_bytes,
                                                    uint32_t bt_base, int items) {
  constexpr int kBt = wgrad_tbuf_bytes(false, NT);
  constexpr int kUnitsO = ((NT + 31) / 32) * 8;        // values of o (8 lanes each) covering round32(NT) channels
  constexpr int kIters = (kUnitsO + 11) / 12;          // 12 groups of 8 lanes in warps 1-3
  constexpr int y_bytes = 4 * kWgradKp * 128;          // dY: 128 channels = 4 chunks
  const int tt = threadIdx.x - 32;
  const int lane = threadIdx.x & 31;
  const int b = tt & 7, b0 = b & 1, b1 = (b >> 1) & 1, b2 = b >> 2;
  // per unit: source offset of pixel 8kk + e (+ 2i: 256 i bytes, slot ^ 2i), Bt offset of channel 4 c4 (+ r: 128 r bytes, slot ^ r)
  uint32_t src[kIters], dst[kIters], sq[kIters], dq[kIters];
  bool ok[kIters];
#pragma unroll
  for (int it = 0; it < kIters; ++it) {
    const int o = (tt >> 3) + 12 * it;
    const int kk = (b1 ^ (o & 1)) | ((b2 ^ ((o >> 1) & 1)) << 1);
    const int c4 = (o >> 3) * 8 + b2 * 4 + b1 * 2 + ((o >> 2) & 1);
    ok[it] = o < kUnitsO && c4 < NT / 4;
    src[it] = y_bytes + (c4 >> 3) * (kWgradKp * 128) + (8 * kk + b0) * 128;
    sq[it] = (c4 & 7) ^ b0;                          // slot of pixel 8kk + e before the ^ 2i
    dst[it] = c4 * 4 * 128;
    dq[it] = (2 * kk + b0) ^ ((c4 & 1) << 2);        // slot of channel 4 c4 before the ^ r
  }
  int stage = 0, tb = 0;
  uint32_t phase = 0, tphase = 0;
  for (int item = blockIdx.x; item < items; item += gridDim.x) {
    const int ks = item % p.ksplits;
    const int blk0 = static_cast<int>((static_cast<long long>(p.px_blocks) * ks) / p.ksplits);
    const int blk1 = static_cast<int>((static_cast<long long>(p.px_blocks) * (ks + 1)) / p.ksplits);
    for (int blk = blk0; blk < blk1; ++blk) {
      mbar_wait(&ctl->full[stage], phase);
      mbar_wait(&ctl->bt_empty[tb], tphase ^ 1);
      const uint32_t sx = stage_base + stage * stage_bytes;
      const uint32_t bt = bt_base + tb * kBt;
#pragma unroll
      for (int it = 0; it < kIters; ++it) {
        if (ok[it]) {
          uint4 v[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) v[i] = lds128(sx + src[it] + 256 * i + ((sq[it] ^ (2 * i)) << 4));
          sts128(bt + dst[it] + ((dq[it] ^ 0) << 4), v[0].x, v[1].x, v[2].x, v[3].x);
          sts128(bt + dst[it] + 128 + ((dq[it] ^ 1) << 4), v[0].y, v[1].y, v[2].y, v[3].y);
          sts128(bt + dst[it] + 256 + ((dq[it] ^ 2) << 4), v[0].z, v[1].z, v[2].z, v[3].z);
          sts128(bt + dst[it] + 384 + ((dq[it] ^ 3) << 4), v[0].w, v[1].w, v[2].w, v[3].w);
        }
      }
      fence_proxy_async_smem();                  // the Bt writes are read by wgmma (async proxy)
      mbar_arrive(&ctl->bt_full[tb]);            // one arrival per transposer thread
      __syncwarp();
      if (lane == 0) mbar_arrive(&ctl->empty[stage]);
      if (++stage == p.stages) { stage = 0; phase ^= 1; }
      tb ^= 1;
      if (tb == 0) tphase ^= 1;
    }
  }
}

// Warps 4-7 (one warpgroup): register-A wgmmas on the dY stage and the Bt tile, fp32 accumulators [2 m64 halves][NT / 2].
// The A fragments of block n+1 are loaded while the wgmmas of block n run (two register sets, fa / fb), except at NT = 160,
// where NT accumulators + 64 fragment registers do not fit in 255 registers: there the loads wait for the wgmmas.
template <int NT>
__device__ __forceinline__ void tc_wgrad_mma(const TcWgradParams& p, SmemCtlW* ctl, uint32_t stage_base, int stage_bytes,
                                             uint32_t bt_base, int items) {
  constexpr int kBt = wgrad_tbuf_bytes(false, NT);
  constexpr bool kDouble = NT <= 136;
  const int et = threadIdx.x - 128;
  const int w = et >> 5, lane = et & 31, g = lane >> 2, t = lane & 3;
  const int taps = p.kh * p.kw;
  // A fragment of k8 step kk, m64 half h: a[0] = (channel n, pixel 8kk + 2t), a[1] = (n + 8, same), a[2] / a[3] = pixel + 1,
  // n = 64h + 16w + g.  Channel n sits in chunk n / 32 = 2h + w / 2, 16-byte group q = 4 (w & 1) + g / 4 (+ 2 for n + 8),
  // word g & 3; pixel 8kk + 2t + e in row 8kk + 2t + e, slot q ^ (2t + e).  Bank argument: over a warp (g, t) the slot takes
  // 8 distinct values (bit 0 = g / 4 ^ e, bits 1-2 = t ^ (2 (w & 1) + hi), hi = 1 for n + 8) and the word g & 3 four more:
  // 32 distinct banks.
  uint32_t aoff[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int hi = r & 1, e = r >> 1;
    const int q = 4 * (w & 1) + (g >> 2) + 2 * hi, px = 2 * t + e;
    aoff[r] = (w >> 1) * (kWgradKp * 128) + px * 128 + ((q ^ px) << 4) + (g & 3) * 4;
  }
  auto load_a = [&](uint32_t (&f)[8][4], uint32_t sy) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
#pragma unroll
        for (int r = 0; r < 4; ++r) f[4 * h + kk][r] = lds32(sy + aoff[r] + h * 2 * (kWgradKp * 128) + kk * 1024);
  };
  int stage = 0, tb = 0;
  uint32_t phase = 0, tphase = 0;
  bool pending = false;   // the previous block's Bt buffer is still to be handed back
  float acc[2][NT / 2];
  uint32_t fa[8][4], fb[8][4];
  // one pixel block: the wgmmas on `cur`, then (while they run) the A fragments of the next block into `nxt`
  auto step = [&](uint32_t (&cur)[8][4], uint32_t (&nxt)[8][4], bool more) {
    mbar_wait(&ctl->bt_full[tb], tphase);
    const uint32_t b_lo = desc_lo(bt_base + tb * kBt);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {   // K-major SW128: advancing K by 8 fp32 = +32 B inside the swizzle atom
      wgmma_rs<NT>(acc[0], cur[kk], desc_of(b_lo + 2 * kk));
      wgmma_rs<NT>(acc[1], cur[4 + kk], desc_of(b_lo + 2 * kk));
    }
    wgmma_commit();
    __syncwarp();
    if (lane == 0) mbar_arrive(&ctl->empty[stage]);   // this block's dY was loaded into registers (and X transposed)
    if (++stage == p.stages) { stage = 0; phase ^= 1; }
    // the previous block's wgmmas are done: its Bt buffer and its fragment registers (nxt) are free
    if constexpr (kDouble) wgmma_wait<1>(); else wgmma_wait<0>();
    if (pending && lane == 0) mbar_arrive(&ctl->bt_empty[tb ^ 1]);
    pending = true;
    tb ^= 1;
    if (tb == 0) tphase ^= 1;
    if (more) {
      mbar_wait(&ctl->full[stage], phase);
      load_a(nxt, stage_base + stage * stage_bytes);
    }
  };
  for (int item = blockIdx.x; item < items; item += gridDim.x) {
    const int tap = item / p.ksplits, ks = item % p.ksplits;
    const int blk0 = static_cast<int>((static_cast<long long>(p.px_blocks) * ks) / p.ksplits);
    const int blk1 = static_cast<int>((static_cast<long long>(p.px_blocks) * (ks + 1)) / p.ksplits);
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
    if (blk0 < blk1) {
      mbar_wait(&ctl->full[stage], phase);
      load_a(fa, stage_base + stage * stage_bytes);
    }
    for (int blk = blk0; blk < blk1; blk += 2) {
      step(fa, kDouble ? fb : fa, blk + 1 < blk1);
      if (blk + 1 == blk1) break;
      step(kDouble ? fb : fa, fa, blk + 2 < blk1);
    }
    wgmma_wait<0>();
    if (pending && lane == 0) mbar_arrive(&ctl->bt_empty[tb ^ 1]);
    pending = false;
    float* dst = p.partial + (static_cast<size_t>(ks) * taps + tap) * 128 * NT;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int j = 0; j < NT / 8; ++j) {
        const int col = 8 * j + 2 * t;
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const int n = 64 * h + 16 * w + g + 8 * rr;   // output channel
          *reinterpret_cast<float2*>(dst + static_cast<size_t>(n) * NT + col) =
              make_float2(acc[h][4 * j + 2 * rr], acc[h][4 * j + 2 * rr + 1]);
        }
      }
    }
  }
}

// The bf16 weight gradient: the consumer warpgroup transposes the pixel-major stage (dY: 128 channels, X: NT channels,
// kWgradKp pixels each, 128-byte swizzled rows of 64 bf16 channels) into K-major swizzled tiles At [128 rows][kWgradKp pixels]
// and Bt [NT rows][kWgradKp pixels] (pixel pairs packed into 32-bit words), then D[n][c] += At * Bt^T.
template <int NT>
__device__ __forceinline__ void tc_wgrad_consumer_bf16(const TcWgradParams& p, SmemCtlW* ctl, uint8_t* smem, int stage_bytes,
                                                       uint8_t* tbase, int items) {
  constexpr int KE = 64;                             // channels per 128-byte source row
  constexpr int E = 2;                               // bytes per element
  constexpr int kTA = kTileM * 128;                  // At: 128 rows of 128 bytes
  constexpr int kTBuf = wgrad_tbuf_bytes(true, NT);
  constexpr int kRows = 128 + NT;
  const int et = threadIdx.x - 128;
  const int w = et >> 5, lane = et & 31;
  constexpr int chunk_bytes = kWgradKp * 128;
  constexpr int y_bytes = (128 / KE) * chunk_bytes;
  constexpr int groups = kWgradKp * E / 16;          // 16-byte K groups per transposed row
  constexpr int nk = kWgradKp / 16;                  // wgmma K steps per pixel block
  const int taps = p.kh * p.kw;
  int stage = 0, tb = 0;
  uint32_t phase = 0;
  float acc[2][NT / 2];
  for (int item = blockIdx.x; item < items; item += gridDim.x) {
    const int tap = item / p.ksplits, ks = item % p.ksplits;
    const int blk0 = static_cast<int>((static_cast<long long>(p.px_blocks) * ks) / p.ksplits);
    const int blk1 = static_cast<int>((static_cast<long long>(p.px_blocks) * (ks + 1)) / p.ksplits);
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
    for (int blk = blk0; blk < blk1; ++blk) {
      mbar_wait(&ctl->full[stage], phase);
      named_bar_sync(1, 128);   // every thread is past the wait of the wgmmas that last read buffer tb
      const uint8_t* sy = smem + stage * stage_bytes;
      const uint8_t* sx = sy + y_bytes;
      uint8_t* ta = tbase + tb * kTBuf;
      uint8_t* tbb = ta + kTA;
      for (int i = et; i < kRows * groups; i += 128) {
        const int g = i / kRows, row = i % kRows;
        const bool is_y = row < 128;
        const int rs = is_y ? row : row - 128;
        const uint8_t* src = (is_y ? sy : sx) + (rs / KE) * chunk_bytes;
        const int cb = (rs % KE) * E;                 // byte of this channel inside a source row
        uint32_t v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int px = g * 8 + 2 * u;
          const uint32_t lo = *reinterpret_cast<const uint16_t*>(src + px * 128 + ((((cb >> 4) ^ (px & 7)) << 4) | (cb & 15)));
          const uint32_t hi = *reinterpret_cast<const uint16_t*>(src + (px + 1) * 128 + ((((cb >> 4) ^ ((px + 1) & 7)) << 4) | (cb & 15)));
          v[u] = lo | (hi << 16);
        }
        uint8_t* dst = (is_y ? ta : tbb) + rs * 128 + ((g ^ (rs & 7)) << 4);
        *reinterpret_cast<uint4*>(dst) = make_uint4(v[0], v[1], v[2], v[3]);
      }
      fence_proxy_async_smem();
      named_bar_sync(1, 128);
      if (lane == 0) mbar_arrive(&ctl->empty[stage]);   // the stage is fully read: TMA may refill it
      const uint32_t a_lo = desc_lo(smem_u32(ta)), b_lo = desc_lo(smem_u32(tbb));
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < nk; ++k) {
        wgmma_ss<NT, true>(acc[0], desc_of(a_lo + 2 * k), desc_of(b_lo + 2 * k));
        wgmma_ss<NT, true>(acc[1], desc_of(a_lo + ((64u * 128u) >> 4) + 2 * k), desc_of(b_lo + 2 * k));
      }
      wgmma_commit();
      wgmma_wait<1>();
      tb ^= 1;
      if (++stage == p.stages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    float* dst = p.partial + (static_cast<size_t>(ks) * taps + tap) * 128 * NT;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int j = 0; j < NT / 8; ++j) {
        const int col = 8 * j + 2 * (lane & 3);
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const int n = 64 * h + 16 * w + (lane >> 2) + 8 * rr;   // output channel
          *reinterpret_cast<float2*>(dst + static_cast<size_t>(n) * NT + col) =
              make_float2(acc[h][4 * j + 2 * rr], acc[h][4 * j + 2 * rr + 1]);
        }
      }
    }
  }
}

template <bool BF16, int NT>
__device__ __forceinline__ void tc_wgrad_role(const TcWgradParams& p, SmemCtlW* ctl, uint8_t* smem, int stage_bytes,
                                              uint8_t* tbase, int items, int warp) {
  if constexpr (BF16) {
    if (warp >= 4) tc_wgrad_consumer_bf16<NT>(p, ctl, smem, stage_bytes, tbase, items);
  } else {
    if (warp >= 4) tc_wgrad_mma<NT>(p, ctl, smem_u32(smem), stage_bytes, smem_u32(tbase), items);
    else tc_wgrad_transposer<NT>(p, ctl, smem_u32(smem), stage_bytes, smem_u32(tbase), items);
  }
}

template <bool BF16>
__device__ __forceinline__ void tc_wgrad_body(const TcWgradParams& p, uint8_t* smem_raw) {
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int KE = BF16 ? 64 : 32;                           // channels per 128-byte row
  constexpr int YCH = 128 / KE;                                // chunks of dY (128 channels)
  constexpr int chunk_bytes = kWgradKp * 128;                  // kWgradKp pixel rows x KE channels
  const int y_bytes = YCH * chunk_bytes;                       // dY: 128 channels
  const int x_bytes = p.c_chunks * chunk_bytes;                // X : c_chunks * KE channels
  const int stage_bytes = y_bytes + x_bytes;
  uint8_t* tbase = smem + p.stages * stage_bytes;              // two transposed operand buffers
  SmemCtlW* ctl = reinterpret_cast<SmemCtlW*>(tbase + 2 * wgrad_tbuf_bytes(BF16, p.n_cols));
  const int items = p.kh * p.kw * p.ksplits;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  pdl_trigger();
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&p.tmY);
    tma_prefetch_desc(&p.tmX);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < p.stages; ++i) {
      mbar_init(&ctl->full[i], 1);
      mbar_init(&ctl->empty[i], BF16 ? 4 : 7);   // one arrival per consumer warp (tf32: and per transposer warp)
    }
    for (int i = 0; i < 2; ++i) {
      mbar_init(&ctl->bt_full[i], 96);   // every transposer thread
      mbar_init(&ctl->bt_empty[i], 4);   // one arrival per MMA warp
    }
    fence_mbar_init();
  }
  pdl_wait();
  __syncthreads();

  if (warp == 0) {
    int stage = 0;
    uint32_t phase = 0;
    for (int item = blockIdx.x; item < items; item += gridDim.x) {
      const int tap = item / p.ksplits, ks = item % p.ksplits;
      const int r = tap / p.kw, s = tap % p.kw;
      const int blk0 = static_cast<int>((static_cast<long long>(p.px_blocks) * ks) / p.ksplits);
      const int blk1 = static_cast<int>((static_cast<long long>(p.px_blocks) * (ks + 1)) / p.ksplits);
      const int ix = p.offx + s, iy = p.offy + r;
      for (int blk = blk0; blk < blk1; ++blk) {
        const int y = blk / p.px_blocks_x;
        const int x0 = (blk % p.px_blocks_x) * kWgradKp;
        int cpx, cx, cpy, cy;
        if (p.stride == 1) {
          cpx = 0; cx = x0 + ix; cpy = 0; cy = y + iy;
        } else {
          cpx = ix & 1; cx = x0 + (ix >> 1); cpy = iy & 1; cy = y + (iy >> 1);
        }
        mbar_wait(&ctl->empty[stage], phase ^ 1);
        uint8_t* sy = smem + stage * stage_bytes;
        if (elect_one()) {
          mbar_expect_tx(&ctl->full[stage], stage_bytes);
          for (int j = 0; j < YCH; ++j) tma_load_3d(sy + j * chunk_bytes, &p.tmY, &ctl->full[stage], j * KE, x0, y);
          for (int j = 0; j < p.c_chunks; ++j)
            tma_load_5d(sy + y_bytes + j * chunk_bytes, &p.tmX, &ctl->full[stage], j * KE, cpx, cx, cpy, cy);
        }
        __syncwarp();
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    switch (p.n_cols) {
      case 32: tc_wgrad_role<BF16, 32>(p, ctl, smem, stage_bytes, tbase, items, warp); break;
      case 64: tc_wgrad_role<BF16, 64>(p, ctl, smem, stage_bytes, tbase, items, warp); break;
      case 96: tc_wgrad_role<BF16, 96>(p, ctl, smem, stage_bytes, tbase, items, warp); break;
      case 128: tc_wgrad_role<BF16, 128>(p, ctl, smem, stage_bytes, tbase, items, warp); break;
      case 136: tc_wgrad_role<BF16, 136>(p, ctl, smem, stage_bytes, tbase, items, warp); break;
      default: tc_wgrad_role<BF16, 160>(p, ctl, smem, stage_bytes, tbase, items, warp); break;
    }
  }
  __syncthreads();
}
__global__ void __launch_bounds__(kNumThreads, 1) tc_wgrad_kernel(const __grid_constant__ TcWgradParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  tc_wgrad_body<false>(p, smem_raw);
}
__global__ void __launch_bounds__(kNumThreads, 1) tc_wgrad_kernel_bf16(const __grid_constant__ TcWgradParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  tc_wgrad_body<true>(p, smem_raw);
}

// ------------------------------------------------------------------------------------------------ host side
static constexpr size_t kMaxSmem = 232448;  // 227 KB

size_t tc_conv_smem_bytes(const TcConvParams& p) {
  const size_t b_bytes = round1024((p.patch ? patch_nt(p.n_mma) : round32(p.n_mma)) * 128);
  if (p.patch)
    return 1024 + p.stages * b_bytes + static_cast<size_t>(p.n_chunks) * kChunkBytes +
           static_cast<size_t>(p.kblocks) * kPatchBytes + sizeof(SmemCtl) + sizeof(PatchCtl);
  return 1024 + p.stages * (kABytes + b_bytes) + static_cast<size_t>(p.n_chunks) * kChunkBytes + sizeof(SmemCtl);
}
size_t tc_wgrad_smem_bytes(const TcWgradParams& p) {
  const size_t chunk = static_cast<size_t>(kWgradKp) * 128;
  const size_t tbuf = wgrad_tbuf_bytes(p.bf16 != 0, p.n_cols);
  return 1024 + p.stages * ((p.bf16 ? 2 : 4) * chunk + static_cast<size_t>(p.c_chunks) * chunk) + 2 * tbuf + sizeof(SmemCtlW);
}

cudaError_t tc_kernels_init() {
  cudaError_t e = cudaFuncSetAttribute(tc_conv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxSmem);
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(tc_conv_kernel_bf16, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxSmem);
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(tc_conv_patch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxSmem);
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(tc_conv_patch_kernel_bf16, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxSmem);
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(tc_wgrad_kernel_bf16, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxSmem);
  if (e != cudaSuccess) return e;
  return cudaFuncSetAttribute(tc_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxSmem);
}

static bool conv_params_ok(const TcConvParams& p) {
  return p.n_mma >= 1 && p.n_mma <= 160 && p.n_chunks == (p.n_mma + 31) / 32 && p.stages >= 1 && p.stages <= 8 &&
         p.kblocks >= 1 && p.nphase >= 0 && p.nphase <= 4 &&
         (p.bw & (p.bw - 1)) == 0 && p.bw * p.bh == kTileM &&
         (!p.patch || (((p.bw == 8 && p.bh == 16) || (p.bw == 16 && p.bh == 8)) && p.kblocks <= kPatchMaxKb && p.kh == 3 && p.kw == 3 && p.stride == 1 && p.nphase == 0));
}

cudaError_t tc_conv_launch(const TcConvParams& p, int num_sms, cudaStream_t s) {
  if (!conv_params_ok(p)) return cudaErrorInvalidValue;
  const int tiles = p.tiles_x * p.tiles_y * (p.nphase > 0 ? p.nphase : 1);
  int grid = tiles < num_sms ? tiles : num_sms;
  if (p.n_split > 1) {
    if (tiles * p.n_split > num_sms) return cudaErrorInvalidValue;
    grid = tiles * p.n_split;   // one CTA per (tile, channel part)
  }
  const size_t smem = tc_conv_smem_bytes(p);
  if (smem > kMaxSmem) return cudaErrorInvalidValue;
  if (p.patch)
    return launch_k(p.bf16 ? tc_conv_patch_kernel_bf16 : tc_conv_patch_kernel, dim3(grid), dim3(kNumThreads), smem, s, 1, p);
  return launch_k(p.bf16 ? tc_conv_kernel_bf16 : tc_conv_kernel, dim3(grid), dim3(kNumThreads), smem, s, 1, p);
}

cudaError_t tc_wgrad_launch(const TcWgradParams& p, cudaStream_t s) {
  const size_t smem = tc_wgrad_smem_bytes(p);
  const bool cols_ok = p.n_cols == 32 || p.n_cols == 64 || p.n_cols == 96 || p.n_cols == 128 || p.n_cols == 136 ||
                       p.n_cols == 160;
  if (smem > kMaxSmem || !cols_ok || p.n_cols > p.c_chunks * (p.bf16 ? 64 : 32) || p.stages < 1 || p.stages > 8)
    return cudaErrorInvalidValue;
  return launch_k(p.bf16 ? tc_wgrad_kernel_bf16 : tc_wgrad_kernel, dim3(p.kh * p.kw * p.ksplits), dim3(kNumThreads), smem, s, 1, p);
}

}  // namespace dip
