// fp32 depthwise 3x3 convolution of the YOLOv11 training step (BASELINE configs[3]), forward / dgrad / wgrad -
// Convs.DWConv (Modules/Convs.cs:108-114, groups = gcd(c1, c2) = c for every use in Yolov11: Head.cs:50 class branch,
// Block.cs:746 Attention.pe).  The YOLOv8 step does not need it; the v11 step's other extra module, the attention core,
// is in attention.cu.  These kernels replace the libtorch autograd kernels behind `loss.backward()` (Utils/Amp.cs:260-286).
// Forward and dgrad run the 4-channel x 4-pixel row kernel when C % 4 == 0 and its weight tile fits, else the scalar
// kernel; wgrad runs the 4- or 1-channel slab partials, then one fold.  Everything is deterministic: reductions run in a
// fixed order (per-slab partials folded in order), no floating-point atomics.  Layouts are the training path's NHWC fp32.
#include <cmath>

#include "common.cuh"

namespace yb {

// ---------------------------------------------------------------------------------------------------------------
// depthwise 3x3, stride 1, pad 1.  x, z, dz, dx: (N, H, W, C);  w: (C, 1, 3, 3) checkpoint layout
// ---------------------------------------------------------------------------------------------------------------
__global__ void dw3x3_forward_kernel(const float* __restrict__ x, const float* __restrict__ w, float* __restrict__ z,
                                     int N, int H, int W, int C, int transpose_taps) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)N * H * W * C;
  if (idx >= total) return;
  const int c = (int)(idx % C);
  size_t p = idx / C;
  const int wx = (int)(p % W);
  p /= W;
  const int hy = (int)(p % H);
  const int n = (int)(p / H);
  float acc = 0.f;
#pragma unroll
  for (int kh = 0; kh < 3; kh++) {
    const int yy = hy + kh - 1;
    if (yy < 0 || yy >= H) continue;
#pragma unroll
    for (int kw = 0; kw < 3; kw++) {
      const int xx = wx + kw - 1;
      if (xx < 0 || xx >= W) continue;
      // dgrad = the same stencil with the taps rotated by 180 degrees
      const int t = transpose_taps ? (2 - kh) * 3 + (2 - kw) : kh * 3 + kw;
      acc = fmaf(x[(((size_t)n * H + yy) * W + xx) * C + c], w[c * 9 + t], acc);
    }
  }
  z[idx] = acc;
}

// 4 channels x 4 adjacent pixels of a row per thread: the 3 x 6 input window is loaded once (18 x 16 B, addresses clamped and
// out-of-image values zeroed afterwards, so that no load is predicated and all are in flight together) and feeds four
// outputs; the weights sit in shared memory as [tap][C].  Same fmaf chain per output element as the scalar kernel above
// (taps in kh, kw order; a zero-padded tap adds 0 * w).  A per-pixel 4-channel kernel needs 9 predicated loads and 36
// scalar weight loads per 4 outputs.
__global__ void __launch_bounds__(256) dw3x3_forward_row4_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                                float* __restrict__ z, int N, int H, int W, int C, int transpose_taps,
                                                                int total) {
  extern __shared__ float dw_sw[];  // [9][C]
  for (int i = threadIdx.x; i < 9 * C; i += blockDim.x) {
    const int t = i / C, c = i - t * C;
    dw_sw[i] = w[c * 9 + (transpose_taps ? 8 - t : t)];
  }
  __syncthreads();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int C4 = C >> 2, WG = (W + 3) >> 2;
  const int c = (idx % C4) * 4;
  int g = idx / C4;
  const int wx0 = (g % WG) * 4;
  g /= WG;
  const int hy = g % H;
  const int n = g / H;
  float4 v[3][6];
#pragma unroll
  for (int kh = 0; kh < 3; kh++) {
    const int yy = hy + kh - 1;
    const int yc = min(max(yy, 0), H - 1);
    const float* row = x + ((size_t)n * H + yc) * W * C + c;
#pragma unroll
    for (int j = 0; j < 6; j++) {
      const int xx = wx0 + j - 1;
      v[kh][j] = __ldg(reinterpret_cast<const float4*>(row + (size_t)min(max(xx, 0), W - 1) * C));
    }
  }
#pragma unroll
  for (int kh = 0; kh < 3; kh++) {
    const int yy = hy + kh - 1;
    const bool vy = yy >= 0 && yy < H;
#pragma unroll
    for (int j = 0; j < 6; j++) {
      const int xx = wx0 + j - 1;
      if (!(vy && xx >= 0 && xx < W)) v[kh][j] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  float4 acc[4];
#pragma unroll
  for (int o = 0; o < 4; o++) acc[o] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int kh = 0; kh < 3; kh++)
#pragma unroll
    for (int kw = 0; kw < 3; kw++) {
      const float4 wt = *reinterpret_cast<const float4*>(dw_sw + (kh * 3 + kw) * C + c);
#pragma unroll
      for (int o = 0; o < 4; o++) {
        const float4 u = v[kh][o + kw];
        acc[o].x = fmaf(u.x, wt.x, acc[o].x);
        acc[o].y = fmaf(u.y, wt.y, acc[o].y);
        acc[o].z = fmaf(u.z, wt.z, acc[o].z);
        acc[o].w = fmaf(u.w, wt.w, acc[o].w);
      }
    }
  float* out = z + (((size_t)n * H + hy) * W + wx0) * C + c;
#pragma unroll
  for (int o = 0; o < 4; o++)
    if (wx0 + o < W) *reinterpret_cast<float4*>(out + (size_t)o * C) = acc[o];
}

// dw[c][t] = sum over pixels dz[p][c] * x[p + tap t][c]: slabs of 256 pixel rows -> partial[slab][t][c]
constexpr int DW_SLAB = 256;
__global__ void __launch_bounds__(256) dw3x3_wgrad_partial_kernel(const float* __restrict__ x, const float* __restrict__ dz,
                                                                 float* __restrict__ partial, int N, int H, int W, int C) {
  __shared__ float red[8][9][32];
  const int cl = threadIdx.x & 31, r = threadIdx.x >> 5;  // 32 channels x 8 row stripes
  const int c = blockIdx.x * 32 + cl;
  const long long rows = (long long)N * H * W;
  const long long r0 = (long long)blockIdx.y * DW_SLAB;
  float acc[9];
#pragma unroll
  for (int t = 0; t < 9; t++) acc[t] = 0.f;
  if (c < C) {
    for (long long p = r0 + r; p < r0 + DW_SLAB && p < rows; p += 8) {
      const int wx = (int)(p % W);
      const long long q = p / W;
      const int hy = (int)(q % H);
      const long long n = q / H;
      const float g = dz[p * C + c];
#pragma unroll
      for (int kh = 0; kh < 3; kh++) {
        const int yy = hy + kh - 1;
        if (yy < 0 || yy >= H) continue;
#pragma unroll
        for (int kw = 0; kw < 3; kw++) {
          const int xx = wx + kw - 1;
          if (xx < 0 || xx >= W) continue;
          acc[kh * 3 + kw] = fmaf(g, x[((n * H + yy) * W + xx) * C + c], acc[kh * 3 + kw]);
        }
      }
    }
  }
#pragma unroll
  for (int t = 0; t < 9; t++) red[r][t][cl] = acc[t];
  __syncthreads();
  if (r == 0 && c < C) {
#pragma unroll
    for (int t = 0; t < 9; t++) {
      float s = 0.f;
      for (int k = 0; k < 8; k++) s += red[k][t][cl];  // fixed order
      partial[((size_t)blockIdx.y * 9 + t) * C + c] = s;
    }
  }
}

// 4 channels per thread, same slabs / stripes / summation order as dw3x3_wgrad_partial_kernel (bit-identical partials):
// 9 + 1 unpredicated 16-byte loads per pixel (clamped addresses, zeroed afterwards) instead of 10 predicated scalar ones
__global__ void __launch_bounds__(256) dw3x3_wgrad_partial4_kernel(const float* __restrict__ x, const float* __restrict__ dz,
                                                                  float* __restrict__ partial, int N, int H, int W, int C) {
  __shared__ float4 red4[8][9][32];
  const int cl = threadIdx.x & 31, r = threadIdx.x >> 5;  // 32 channel quads x 8 row stripes
  const int c = (blockIdx.x * 32 + cl) * 4;
  const long long rows = (long long)N * H * W;
  const long long r0 = (long long)blockIdx.y * DW_SLAB;
  float4 acc[9];
#pragma unroll
  for (int t = 0; t < 9; t++) acc[t] = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c < C) {
    for (long long p = r0 + r; p < r0 + DW_SLAB && p < rows; p += 8) {
      const int wx = (int)(p % W);
      const long long q = p / W;
      const int hy = (int)(q % H);
      const long long n = q / H;
      const float4 g = __ldg(reinterpret_cast<const float4*>(dz + p * C + c));
      float4 u[9];
#pragma unroll
      for (int kh = 0; kh < 3; kh++) {
        const int yc = min(max(hy + kh - 1, 0), H - 1);
#pragma unroll
        for (int kw = 0; kw < 3; kw++) {
          const int xc = min(max(wx + kw - 1, 0), W - 1);
          u[kh * 3 + kw] = __ldg(reinterpret_cast<const float4*>(x + ((n * H + yc) * W + xc) * C + c));
        }
      }
#pragma unroll
      for (int kh = 0; kh < 3; kh++) {
        const int yy = hy + kh - 1;
#pragma unroll
        for (int kw = 0; kw < 3; kw++) {
          const int xx = wx + kw - 1;
          const int t = kh * 3 + kw;
          if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;  // the scalar kernel skips these taps: keep -0 / NaN behaviour
          acc[t].x = fmaf(g.x, u[t].x, acc[t].x);
          acc[t].y = fmaf(g.y, u[t].y, acc[t].y);
          acc[t].z = fmaf(g.z, u[t].z, acc[t].z);
          acc[t].w = fmaf(g.w, u[t].w, acc[t].w);
        }
      }
    }
  }
#pragma unroll
  for (int t = 0; t < 9; t++) red4[r][t][cl] = acc[t];
  __syncthreads();
  if (r == 0 && c < C) {
#pragma unroll
    for (int t = 0; t < 9; t++) {
      float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int k = 0; k < 8; k++) {  // fixed order
        const float4 e = red4[k][t][cl];
        sum.x += e.x; sum.y += e.y; sum.z += e.z; sum.w += e.w;
      }
      *reinterpret_cast<float4*>(partial + ((size_t)blockIdx.y * 9 + t) * C + c) = sum;
    }
  }
}

// fold of the slab partials with 8 lanes per (tap, channel): lane y adds slabs y, y + 8, ... in order, lanes added in order
// (one thread walking 400 slabs serially would be a long dependent-load chain)
__global__ void __launch_bounds__(256) dw3x3_wgrad_fold8_kernel(const float* __restrict__ partial, float* __restrict__ dw, int slabs, int C) {
  __shared__ float f[8][32];
  const int i = blockIdx.x * 32 + threadIdx.x;  // (t, c)
  float a = 0.f;
  if (i < 9 * C)
    for (int k = threadIdx.y; k < slabs; k += 8) a += partial[(size_t)k * 9 * C + i];
  f[threadIdx.y][threadIdx.x] = a;
  __syncthreads();
  if (threadIdx.y != 0 || i >= 9 * C) return;
  float sum = 0.f;
  for (int k = 0; k < 8; k++) sum += f[k][threadIdx.x];
  const int t = i / C, c = i - t * C;
  dw[c * 9 + t] = sum;
}

static bool dw_row4_ok(int N, int H, int W, int C, const void* a, const void* b) {
  return C % 4 == 0 && (size_t)9 * C * sizeof(float) <= 48 * 1024 && (size_t)N * H * ((W + 3) / 4) * (C / 4) < ((size_t)1 << 31) &&
         !(((uintptr_t)a | (uintptr_t)b) & 15);
}
int dwconv3x3_forward_f32(const float* x, const float* w, int N, int H, int W, int C, float* z, cudaStream_t s) {
  const size_t total = (size_t)N * H * W * C;
  if (dw_row4_ok(N, H, W, C, x, z)) {
    const int tot = N * H * ((W + 3) / 4) * (C / 4);
    dw3x3_forward_row4_kernel<<<(unsigned)((tot + 255) / 256), 256, (size_t)9 * C * sizeof(float), s>>>(x, w, z, N, H, W, C, 0, tot);
  } else
    dw3x3_forward_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(x, w, z, N, H, W, C, 0);
  YB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int dwconv3x3_backward_f32(const float* x, const float* dz, const float* w, int N, int H, int W, int C, float* dx, float* dw,
                           cudaStream_t s) {
  const size_t total = (size_t)N * H * W * C;
  if (dw_row4_ok(N, H, W, C, dz, dx)) {
    const int tot = N * H * ((W + 3) / 4) * (C / 4);
    dw3x3_forward_row4_kernel<<<(unsigned)((tot + 255) / 256), 256, (size_t)9 * C * sizeof(float), s>>>(dz, w, dx, N, H, W, C, 1, tot);
  } else
    dw3x3_forward_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(dz, w, dx, N, H, W, C, 1);
  YB_CUDA_CHECK(cudaGetLastError());
  const long long rows = (long long)N * H * W;
  const int slabs = (int)((rows + DW_SLAB - 1) / DW_SLAB);
  float* partial = nullptr;
  YB_CUDA_CHECK(cudaMallocAsync((void**)&partial, (size_t)slabs * 9 * C * sizeof(float), s));
  if (C % 4 == 0 && !((uintptr_t)x & 15) && !((uintptr_t)dz & 15))
    dw3x3_wgrad_partial4_kernel<<<dim3((C / 4 + 31) / 32, slabs), 256, 0, s>>>(x, dz, partial, N, H, W, C);
  else
    dw3x3_wgrad_partial_kernel<<<dim3((C + 31) / 32, slabs), 256, 0, s>>>(x, dz, partial, N, H, W, C);
  dw3x3_wgrad_fold8_kernel<<<(9 * C + 31) / 32, dim3(32, 8), 0, s>>>(partial, dw, slabs, C);
  cudaError_t ce = cudaGetLastError();
  cudaFreeAsync(partial, s);
  YB_CUDA_CHECK(ce);
  return 0;
}

}  // namespace yb

using namespace yb;

extern "C" {

int32_t yb_dwconv3x3_forward_f32(const float* x, const float* w, int32_t n, int32_t height, int32_t width, int32_t channels,
                                 float* z, void* stream) {
  if (!x || !w || !z || n <= 0 || height <= 0 || width <= 0 || channels <= 0) { set_error("yb_dwconv3x3_forward_f32: bad argument"); return YB_ERR_INVALID_ARG; }
  if (!have_device("yb_dwconv3x3_forward_f32")) return YB_ERR_NO_DEVICE;
  return dwconv3x3_forward_f32(x, w, n, height, width, channels, z, (cudaStream_t)stream);
}

int32_t yb_dwconv3x3_backward_f32(const float* x, const float* dz, const float* w, int32_t n, int32_t height, int32_t width,
                                  int32_t channels, float* dx, float* dw, void* stream) {
  if (!x || !dz || !w || !dx || !dw || n <= 0 || height <= 0 || width <= 0 || channels <= 0) { set_error("yb_dwconv3x3_backward_f32: bad argument"); return YB_ERR_INVALID_ARG; }
  if (!have_device("yb_dwconv3x3_backward_f32")) return YB_ERR_NO_DEVICE;
  return dwconv3x3_backward_f32(x, dz, w, n, height, width, channels, dx, dw, (cudaStream_t)stream);
}

}  // extern "C"
