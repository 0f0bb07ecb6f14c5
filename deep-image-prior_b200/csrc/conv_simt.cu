// Exact-fp32 CUDA-core convolutions (precision mode "fp32"): same operand layouts and semantics as the wgmma
// kernels in conv_tc.cu, FMA arithmetic in IEEE fp32.  Used for the parity tier that must not see TF32 rounding
// (SURVEY.md section 7.4, P2) and as the on-device cross-check of the tensor-core path.
// Reference semantics: torch.nn.Conv2d forward / backward (models/common.py:120).
#include "kernels.cuh"

namespace dip {

// D[y][x][n] = bias[n] + sum_{r,s,c} A'[y*stride+offy+r][x*stride+offx+s][c] * Wp[tap][n][c]   (OOB reads = 0), where
// A' is A dilated by `dil`: A'[iy][ix] = A[iy / dil][ix / dil] when dil divides both, else 0.  Dilation 2 with stride 1
// is the input gradient of a stride-2 conv, read from dY at its own resolution.
// Block: 16 consecutive output pixels of one row x all n_rows outputs (thread = output channel).
static constexpr int kSimtPx = 16;
__global__ void __launch_bounds__(160) k_simt_conv(SimtConvArgs a) {
  pdl_enter();
  __shared__ __align__(16) float As[32][kSimtPx];  // [c][px]
  __shared__ float Ws[160][33];                    // [n][c] (+1 pad)
  const int sh = a.dil >> 1;                       // dil = 1 or 2: log2(dil), and the mask of an odd coordinate
  const int n = threadIdx.x;
  const int xb = blockIdx.x * kSimtPx;
  const int y = blockIdx.y;
  float acc[kSimtPx];
#pragma unroll
  for (int i = 0; i < kSimtPx; ++i) acc[i] = 0.f;
  for (int r = 0; r < a.kh; ++r) {
    for (int s = 0; s < a.kw; ++s) {
      const int tap = r * a.kw + s;
      const int iy = y * a.stride + a.offy + r;
      for (int c0 = 0; c0 < a.c_pad; c0 += 32) {
        __syncthreads();
        for (int i = threadIdx.x; i < 32 * kSimtPx; i += blockDim.x) {
          const int c = i & 31, px = i >> 5;
          const int ix = (xb + px) * a.stride + a.offx + s;
          float v = 0.f;
          if (iy >= 0 && (iy >> sh) < a.a_h && ix >= 0 && (ix >> sh) < a.a_w && ((iy | ix) & sh) == 0 && c0 + c < a.a_c)
            v = a.A[(static_cast<long long>(iy >> sh) * a.a_w + (ix >> sh)) * a.a_ld + c0 + c];
          As[c][px] = v;
        }
        for (int i = threadIdx.x; i < a.n_rows * 32; i += blockDim.x) {
          const int c = i & 31, nn = i >> 5;
          Ws[nn][c] = a.Wp[(static_cast<long long>(tap) * a.n_rows + nn) * a.c_pad + c0 + c];
        }
        __syncthreads();
        if (n < a.n_rows) {
#pragma unroll 8
          for (int c = 0; c < 32; ++c) {
            const float w = Ws[n][c];
            const float4* ap = reinterpret_cast<const float4*>(&As[c][0]);
#pragma unroll
            for (int q = 0; q < kSimtPx / 4; ++q) {
              const float4 av = ap[q];
              acc[4 * q + 0] = fmaf(av.x, w, acc[4 * q + 0]);
              acc[4 * q + 1] = fmaf(av.y, w, acc[4 * q + 1]);
              acc[4 * q + 2] = fmaf(av.z, w, acc[4 * q + 2]);
              acc[4 * q + 3] = fmaf(av.w, w, acc[4 * q + 3]);
            }
          }
        }
      }
    }
  }
  if (n < a.d_c && y < a.d_h) {
    const float b = a.bias != nullptr ? a.bias[n] : 0.f;
    for (int px = 0; px < kSimtPx; ++px)
      if (xb + px < a.d_w) a.D[(static_cast<long long>(y) * a.d_w + xb + px) * a.d_ld + n] = acc[px] + b;
  }
}
void launch_simt_conv(SimtConvArgs a, cudaStream_t s) {
  dim3 grid((a.d_w + kSimtPx - 1) / kSimtPx, a.d_h);
  launch_k(k_simt_conv, dim3(grid), dim3(160), 0, s, 1, a);
}

// partial[ks][tap][n][c] = sum over the rows of split ks of dY[y][x][n] * X[y*stride+offy+r][x*stride+offx+s][c]
// Block: (tap, group of 8 output channels, split); thread = input channel c.
__global__ void __launch_bounds__(160) k_simt_wgrad(SimtWgradArgs a) {
  pdl_enter();
  const int tap = blockIdx.x, ng = blockIdx.y, ks = blockIdx.z;
  const int r = tap / a.kw, s = tap % a.kw;
  const int c = threadIdx.x;
  const int y0 = static_cast<int>((static_cast<long long>(a.h) * ks) / a.ksplits);
  const int y1 = static_cast<int>((static_cast<long long>(a.h) * (ks + 1)) / a.ksplits);
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  for (int y = y0; y < y1; ++y) {
    const int iy = y * a.stride + a.offy + r;
    if (iy < 0 || iy >= a.x_h) continue;
    for (int x = 0; x < a.w; ++x) {
      const int ix = x * a.stride + a.offx + s;
      if (ix < 0 || ix >= a.x_w) continue;
      float xv = 0.f;
      if (c < a.x_c) xv = a.X[(static_cast<long long>(iy) * a.x_w + ix) * a.x_ld + c];
      const float4* gp = reinterpret_cast<const float4*>(a.dY + (static_cast<long long>(y) * a.w + x) * (a.dy_ld > 0 ? a.dy_ld : 128) + ng * 8);
      const float4 g0 = gp[0], g1 = gp[1];
      acc[0] = fmaf(g0.x, xv, acc[0]); acc[1] = fmaf(g0.y, xv, acc[1]);
      acc[2] = fmaf(g0.z, xv, acc[2]); acc[3] = fmaf(g0.w, xv, acc[3]);
      acc[4] = fmaf(g1.x, xv, acc[4]); acc[5] = fmaf(g1.y, xv, acc[5]);
      acc[6] = fmaf(g1.z, xv, acc[6]); acc[7] = fmaf(g1.w, xv, acc[7]);
    }
  }
  if (c < a.c_pad) {
    const int taps = a.kh * a.kw;
    for (int i = 0; i < 8; ++i)
      a.partial[((static_cast<long long>(ks) * taps + tap) * 128 + ng * 8 + i) * a.c_pad + c] = acc[i];
  }
}
void launch_simt_wgrad(SimtWgradArgs a, cudaStream_t s) {
  dim3 grid(a.kh * a.kw, a.n > 0 ? (a.n + 7) / 8 : 16, a.ksplits);   // output channels in groups of 8 (widths are multiples of 8)
  launch_k(k_simt_wgrad, dim3(grid), dim3(160), 0, s, 1, a);
}

}  // namespace dip
