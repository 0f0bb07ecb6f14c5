// Host-side descriptors for the wgmma implicit-GEMM convolution kernels (conv_tc.cu).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace dip {

// Implicit-GEMM forward/dgrad conv:  D[pixel][n] = sum_{tap, c} A[pixel (+) tap][c] * Wp[tap][n][c]  (+ bias[n])
//   A  : NHWC activation (fp32, or its bf16 twin when bf16 = 1) seen through a 5-D tensor map (C, px, X, py, Y)   (parity
//        dims px/py have extent 1 for stride-1 convs and 2 for stride-2 convs; out-of-bounds coordinates read as zero)
//   Wp : packed weights [tap][n_rows][c_pad] (fp32 or bf16), K-major, through a 2-D map (c_pad, taps*n_rows)
//   D  : NHWC fp32 output through a 3-D map (C_out, W_out, H_out); partial tiles and channels >= C_out are clipped by TMA.
struct TcConvParams {
  CUtensorMap tmA;
  CUtensorMap tmB;
  CUtensorMap tmD;
  int tiles_x, tiles_y;    // output tile grid
  int bw, bh;              // tile = bw x bh output pixels, bw*bh == 128
  int out_w, out_h;        // valid output extent (for masked statistics)
  int kh, kw;              // filter taps
  int stride;              // 1 or 2 (spatial stride of A reads)
  int offx, offy;          // input coordinate of tap (0,0) for output pixel (0,0)
  int bf16;                // 1: bf16 operands: A / Wp are bf16, a K block is 64 channels (still 128 bytes), K = 16 per wgmma
  int kblocks;             // K blocks (128-byte operand rows: 32 fp32 or 64 bf16 channels) per tap
  int n_mma;               // output channels of this CTA (multiple of 16, <= 160): all of them, or N / n_split; the wgmma N is
                           // n_mma rounded up to 32 (columns past n_mma are never stored or counted)
  int n_chunks;            // output 32-channel chunks written (ceil(n_mma/32))
  int stages;              // smem pipeline depth
  int n_split;             // 1, 2 or 4 CTAs per pixel tile, each computing n_mma = N / n_split output channels (small levels)
  // Stride-2 input gradient as its 4 sub-pixel phases in ONE launch (nphase = 4, per-tap mode): output pixel (2i+a, 2j+b)
  // of the padded input gradient only receives the taps r = a (mod 2), s = b (mod 2), i.e. a (2-a) x (2-b) stride-1
  // correlation over dY.  Work item = (phase, tile of the (h+1) x (w+1) phase grid); tmD is then the 5-D parity view
  // (C, px, X, py, Y) of the padded gradient buffer and the tile is stored at parity (opx, opy).  nphase = 0: one phase
  // described by kh / kw / offx / offy above, 3-D tmD.
  int nphase;
  struct Phase { int kh, kw, offx, offy, tap0, opx, opy; } phs[4];   // tap0: first packed weight tap of the phase
  int n_valid;             // output channels that exist (bias / statistics are only read / written below it); 0: all n_mma * n_split
  const float* bias;       // [n_valid] or nullptr
  double* stats;           // [2][stats_ld] per-channel sum / sum of squares (fp64 atomics) or nullptr
  int stats_ld;
  // patch = 1: the stride-1 3x3 path (tc_conv_patch_kernel), tiles bw x bh = 8 x 16 or 16 x 8.  Per tile and K block one
  // (bh + 2) x (bw + 2) pixel patch feeds all nine taps.  tmA is then the 4-D map (channels of one 16-byte group, X, Y,
  // group) of the activation with box {group, bw + 2, bh + 2, 8}: TMA writes the patch as [group][patch row][patch col][16 B].
  int patch;
};
// geometry of the patch path (tc_conv_patch_kernel)
static constexpr int kPatchPlane = 180 * 16;   // one 16-byte channel group of a (bh + 2) x (bw + 2) = 180 pixel patch (2880 B)
static constexpr int kPatchMaxKb = 8;          // K blocks (resident patches) per tile at most
static constexpr int kPatchBytes = 8 * kPatchPlane;                    // one K block: 128 bytes per pixel (23040 B)

// Weight-gradient GEMM:  dW[tap][n][c] = sum_{pixels} dY[pixel][n] * X[pixel (+) tap][c]
//   dY : NHWC [H][W][N] (fp32 or bf16 twin; N <= 128 output channels, channels >= N read as zero) through a 3-D map (N, W, H)
//   X  : conv input through the same 5-D view as in TcConvParams
//   A work item is one filter tap and one split-K range of pixel blocks (kh * kw * ksplits items); it writes its own
//   slice of partials [ksplit][tap][128][n_cols], which a follow-up kernel sums in a fixed order -- the gradient does not
//   depend on the order in which work items finish (fp32 atomics here made runs drift apart over thousands of steps).
// pixels per K block of the weight-gradient GEMM (TMA box width; one transposed 128-byte row holds 32 fp32 pixels).  A row
// shorter than a multiple of 32 reads zero-filled dY past its end, which adds nothing.
static constexpr int kWgradKp = 32;
struct TcWgradParams {
  CUtensorMap tmY;
  CUtensorMap tmX;
  float* partial;          // [ksplits][kh*kw][128][n_cols], every element written by the kernel
  int kh, kw, stride, offx, offy;
  int px_blocks_x;         // ceil(W / kWgradKp)
  int px_blocks;           // total pixel blocks = H * px_blocks_x
  int bf16;                // 1: dY / X are bf16 (chunks of 64 channels, K = 16 pixels per wgmma)
  int c_chunks;            // 128-byte channel chunks of X (32 fp32 / 64 bf16 channels each)
  int n_cols;              // wgmma N = accumulator columns per tap = row stride of `partial`: 32, 64, 96, 128, 136 or 160
                           // (<= the channels of the X chunks; channels past C are zero in X, so their columns are zero)
  int ksplits;             // work items per filter tap
  int stages;
};

size_t tc_conv_smem_bytes(const TcConvParams& p);
size_t tc_wgrad_smem_bytes(const TcWgradParams& p);
cudaError_t tc_conv_launch(const TcConvParams& p, int num_sms, cudaStream_t s);
cudaError_t tc_wgrad_launch(const TcWgradParams& p, cudaStream_t s);
cudaError_t tc_kernels_init();

}  // namespace dip
