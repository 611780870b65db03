// fp32 parity kernels of the YOLOv11 training step (BASELINE configs[3]) that the YOLOv8 step does not need:
//   * depthwise 3x3 convolution, forward / dgrad / wgrad  - Convs.DWConv (Modules/Convs.cs:108-114, groups =
//     gcd(c1, c2) = c for every use in Yolov11: Head.cs:50 class branch, Block.cs:746 Attention.pe)
//   * attention core softmax(q^T k * scale) v, forward / backward  - Block.Attention.forward (Block.cs:785-809)
// They replace the libtorch autograd kernels behind `loss.backward()` (Utils/Amp.cs:260-286) for these modules.
// Everything is deterministic: reductions run in a fixed order (per-slab partials folded sequentially, per-row
// sequential sums), no floating-point atomics.  Layouts are the training path's NHWC fp32 (train.py).
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

// 4 channels per thread (16-byte loads / stores, 32-bit index math); same per-element tap order as the scalar kernel
__global__ void __launch_bounds__(256) dw3x3_forward4_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                            float* __restrict__ z, int N, int H, int W, int C, int transpose_taps,
                                                            int total4) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total4) return;
  const int C4 = C >> 2;
  const int c = (idx % C4) * 4;
  int p = idx / C4;
  const int wx = p % W;
  p /= W;
  const int hy = p % H;
  const int n = p / H;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
  for (int kh = 0; kh < 3; kh++) {
    const int yy = hy + kh - 1;
    if (yy < 0 || yy >= H) continue;
#pragma unroll
    for (int kw = 0; kw < 3; kw++) {
      const int xx = wx + kw - 1;
      if (xx < 0 || xx >= W) continue;
      const int t = transpose_taps ? (2 - kh) * 3 + (2 - kw) : kh * 3 + kw;
      const float4 v = *reinterpret_cast<const float4*>(x + (((size_t)n * H + yy) * W + xx) * C + c);
      a0 = fmaf(v.x, w[c * 9 + t], a0);
      a1 = fmaf(v.y, w[(c + 1) * 9 + t], a1);
      a2 = fmaf(v.z, w[(c + 2) * 9 + t], a2);
      a3 = fmaf(v.w, w[(c + 3) * 9 + t], a3);
    }
  }
  *reinterpret_cast<float4*>(z + (size_t)idx * 4) = make_float4(a0, a1, a2, a3);
}

// 4 channels x 4 adjacent pixels of a row per thread: the 3 x 6 input window is loaded once (18 x 16 B, addresses clamped and
// out-of-image values zeroed afterwards, so that no load is predicated and all are in flight together) and feeds four
// outputs; the weights sit in shared memory as [tap][C].  Same fmaf chain per output element as the kernels above (taps
// in kh, kw order; a zero-padded tap adds 0 * w).  The per-pixel kernel above needs 9 predicated loads and 36 scalar
// weight loads per 4 outputs.
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

__global__ void dw3x3_wgrad_fold_kernel(const float* __restrict__ partial, float* __restrict__ dw, int slabs, int C) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // (t, c)
  if (i >= 9 * C) return;
  const int t = i / C, c = i - t * C;
  float s = 0.f;
  for (int k = 0; k < slabs; k++) s += partial[((size_t)k * 9 + t) * C + c];
  dw[c * 9 + t] = s;
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
  } else if (C % 4 == 0 && total / 4 < ((size_t)1 << 31) && !((uintptr_t)x & 15) && !((uintptr_t)z & 15))
    dw3x3_forward4_kernel<<<(unsigned)((total / 4 + 255) / 256), 256, 0, s>>>(x, w, z, N, H, W, C, 0, (int)(total / 4));
  else
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
  } else if (C % 4 == 0 && total / 4 < ((size_t)1 << 31) && !((uintptr_t)dz & 15) && !((uintptr_t)dx & 15))
    dw3x3_forward4_kernel<<<(unsigned)((total / 4 + 255) / 256), 256, 0, s>>>(dz, w, dx, N, H, W, C, 1, (int)(total / 4));
  else
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

// ---------------------------------------------------------------------------------------------------------------
// attention core.  q, k: (B, N, nh, kd); v, out, dout: (B, N, nh, hd); one block per (row, head, image)
// ---------------------------------------------------------------------------------------------------------------
constexpr int AT_THREADS = 128;

__device__ __forceinline__ float block_max(float v, float* sh) {
  for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = sh[0];
  for (int i = 1; i < AT_THREADS / 32; i++) r = fmaxf(r, sh[i]);
  __syncthreads();
  return r;
}
__device__ __forceinline__ float block_sum(float v, float* sh) {
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = sh[0];
  for (int i = 1; i < AT_THREADS / 32; i++) r += sh[i];  // fixed order
  __syncthreads();
  return r;
}

// forward: out_i = sum_j softmax_j(scale q_i.k_j) v_j; also the row statistics (max, sum) for the backward pass
__global__ void __launch_bounds__(AT_THREADS) attn_forward_kernel(const float* __restrict__ q, const float* __restrict__ k,
                                                                  const float* __restrict__ v, float* __restrict__ out,
                                                                  float* __restrict__ row_max, float* __restrict__ row_sum,
                                                                  int N, int nh, int kd, int hd, float scale) {
  extern __shared__ float sm[];  // p[N] | qrow[kd]
  float* p = sm;
  float* qrow = sm + N;
  __shared__ float red[AT_THREADS / 32];
  const int i = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const size_t qk_stride = (size_t)nh * kd, v_stride = (size_t)nh * hd;
  const float* qi = q + ((size_t)b * N + i) * qk_stride + (size_t)h * kd;
  for (int d = threadIdx.x; d < kd; d += AT_THREADS) qrow[d] = qi[d];
  __syncthreads();
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < N; j += AT_THREADS) {
    const float* kj = k + ((size_t)b * N + j) * qk_stride + (size_t)h * kd;
    float s = 0.f;
    for (int d = 0; d < kd; d++) s = fmaf(qrow[d], kj[d], s);
    s *= scale;
    p[j] = s;
    mx = fmaxf(mx, s);
  }
  mx = block_max(mx, red);
  float sum = 0.f;
  for (int j = threadIdx.x; j < N; j += AT_THREADS) {
    const float e = expf(p[j] - mx);
    p[j] = e;
    sum += e;
  }
  sum = block_sum(sum, red);
  const float inv = 1.0f / sum;
  for (int d = threadIdx.x; d < hd; d += AT_THREADS) {
    const float* vd = v + (size_t)b * N * v_stride + (size_t)h * hd + d;
    float o = 0.f;
    for (int j = 0; j < N; j++) o = fmaf(p[j], vd[(size_t)j * v_stride], o);
    out[((size_t)b * N + i) * v_stride + (size_t)h * hd + d] = o * inv;
  }
  if (threadIdx.x == 0 && row_max) {
    row_max[((size_t)b * nh + h) * N + i] = mx;
    row_sum[((size_t)b * nh + h) * N + i] = sum;
  }
}

// backward pass A, per query row i: D_i = sum_j p_ij dP_ij, dS_ij = p_ij (dP_ij - D_i), dQ_i = scale sum_j dS_ij k_j
__global__ void __launch_bounds__(AT_THREADS) attn_backward_q_kernel(const float* __restrict__ q, const float* __restrict__ k,
                                                                     const float* __restrict__ v, const float* __restrict__ dout,
                                                                     const float* __restrict__ row_max, const float* __restrict__ row_sum,
                                                                     float* __restrict__ row_d, float* __restrict__ dq, int N, int nh,
                                                                     int kd, int hd, float scale) {
  extern __shared__ float sm[];  // ds[N] | qrow[kd] | dorow[hd]
  float* ds = sm;
  float* qrow = sm + N;
  float* dorow = qrow + kd;
  __shared__ float red[AT_THREADS / 32];
  const int i = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const size_t qk_stride = (size_t)nh * kd, v_stride = (size_t)nh * hd;
  const size_t st = ((size_t)b * nh + h) * N + i;
  const float mx = row_max[st], inv = 1.0f / row_sum[st];
  for (int d = threadIdx.x; d < kd; d += AT_THREADS) qrow[d] = q[((size_t)b * N + i) * qk_stride + (size_t)h * kd + d];
  for (int d = threadIdx.x; d < hd; d += AT_THREADS) dorow[d] = dout[((size_t)b * N + i) * v_stride + (size_t)h * hd + d];
  __syncthreads();
  float dsum = 0.f;
  for (int j = threadIdx.x; j < N; j += AT_THREADS) {
    const float* kj = k + ((size_t)b * N + j) * qk_stride + (size_t)h * kd;
    const float* vj = v + ((size_t)b * N + j) * v_stride + (size_t)h * hd;
    float s = 0.f, dp = 0.f;
    for (int d = 0; d < kd; d++) s = fmaf(qrow[d], kj[d], s);
    for (int d = 0; d < hd; d++) dp = fmaf(dorow[d], vj[d], dp);
    const float pj = expf(s * scale - mx) * inv;
    ds[j] = pj;  // p for now; dP is recomputed below (the score row holds N floats only)
    dsum = fmaf(pj, dp, dsum);
  }
  const float D = block_sum(dsum, red);
  for (int j = threadIdx.x; j < N; j += AT_THREADS) {
    const float* vj = v + ((size_t)b * N + j) * v_stride + (size_t)h * hd;
    float dp = 0.f;
    for (int d = 0; d < hd; d++) dp = fmaf(dorow[d], vj[d], dp);
    ds[j] = ds[j] * (dp - D);
  }
  __syncthreads();
  for (int d = threadIdx.x; d < kd; d += AT_THREADS) {
    const float* kd_ = k + (size_t)b * N * qk_stride + (size_t)h * kd + d;
    float a = 0.f;
    for (int j = 0; j < N; j++) a = fmaf(ds[j], kd_[(size_t)j * qk_stride], a);
    dq[((size_t)b * N + i) * qk_stride + (size_t)h * kd + d] = a * scale;
  }
  if (threadIdx.x == 0) row_d[st] = D;
}

// backward pass B, per key row j: dV_j = sum_i p_ij dO_i, dK_j = scale sum_i dS_ij q_i
__global__ void __launch_bounds__(AT_THREADS) attn_backward_kv_kernel(const float* __restrict__ q, const float* __restrict__ k,
                                                                      const float* __restrict__ v, const float* __restrict__ dout,
                                                                      const float* __restrict__ row_max, const float* __restrict__ row_sum,
                                                                      const float* __restrict__ row_d, float* __restrict__ dk,
                                                                      float* __restrict__ dv, int N, int nh, int kd, int hd, float scale) {
  extern __shared__ float sm[];  // p[N] | ds[N] | krow[kd] | vrow[hd]
  float* p = sm;
  float* ds = sm + N;
  float* krow = ds + N;
  float* vrow = krow + kd;
  const int j = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const size_t qk_stride = (size_t)nh * kd, v_stride = (size_t)nh * hd;
  for (int d = threadIdx.x; d < kd; d += AT_THREADS) krow[d] = k[((size_t)b * N + j) * qk_stride + (size_t)h * kd + d];
  for (int d = threadIdx.x; d < hd; d += AT_THREADS) vrow[d] = v[((size_t)b * N + j) * v_stride + (size_t)h * hd + d];
  __syncthreads();
  for (int i = threadIdx.x; i < N; i += AT_THREADS) {
    const float* qi = q + ((size_t)b * N + i) * qk_stride + (size_t)h * kd;
    const float* doi = dout + ((size_t)b * N + i) * v_stride + (size_t)h * hd;
    const size_t st = ((size_t)b * nh + h) * N + i;
    float s = 0.f, dp = 0.f;
    for (int d = 0; d < kd; d++) s = fmaf(qi[d], krow[d], s);
    for (int d = 0; d < hd; d++) dp = fmaf(doi[d], vrow[d], dp);
    const float pij = expf(s * scale - row_max[st]) / row_sum[st];
    p[i] = pij;
    ds[i] = pij * (dp - row_d[st]);
  }
  __syncthreads();
  for (int d = threadIdx.x; d < hd; d += AT_THREADS) {
    const float* dod = dout + (size_t)b * N * v_stride + (size_t)h * hd + d;
    float a = 0.f;
    for (int i = 0; i < N; i++) a = fmaf(p[i], dod[(size_t)i * v_stride], a);
    dv[((size_t)b * N + j) * v_stride + (size_t)h * hd + d] = a;
  }
  for (int d = threadIdx.x; d < kd; d += AT_THREADS) {
    const float* qd = q + (size_t)b * N * qk_stride + (size_t)h * kd + d;
    float a = 0.f;
    for (int i = 0; i < N; i++) a = fmaf(ds[i], qd[(size_t)i * qk_stride], a);
    dk[((size_t)b * N + j) * qk_stride + (size_t)h * kd + d] = a * scale;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Tiled attention (the path that runs for the network's shapes: N = 400 tokens at 640 x 640, kd = 32, hd = 64).
// The row kernels above launch one CTA per (token, head, image) and every CTA streams the head's whole K and V from
// L2 (25 600 CTAs x 150 KB for one YOLOv11s layer at batch 16).  Here a CTA owns a tile of
// AT_T = 16 tokens of one (head, image) and keeps the head's K and V (or Q and dO) in shared memory:
//   row strides kd + 1 / hd + 1 make both access patterns - lanes over tokens (score / dP dot products) and lanes
//   over channels (P.V, dS.K accumulations) - bank-conflict free;  8 warps, two token rows per warp share every
//   shared-memory operand they read.  Same arithmetic order per output as the row kernels (sequential over the
//   reduction index), same saved statistics.
// ---------------------------------------------------------------------------------------------------------------
constexpr int AT_T = 16;
constexpr int ATT_THREADS = 256;  // 8 warps x 2 rows

__device__ __forceinline__ float warp_max(float v) {
  for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// rows of one head of a (B, N, nh, dim) tensor -> shared memory with row stride `ld` (dim a multiple of 4, 16-byte aligned
// rows in global memory).  Eight independent 16-byte loads are in flight per thread: with one CTA of 8 warps per SM a
// load-store loop of scalar loads would expose the full L2 latency per element.
__device__ __forceinline__ void load_head(float* dst, const float* src, int b, int h, int N, int nh, int dim, int ld, int row0,
                                          int rows) {
  constexpr int U = 8;
  const int d4 = dim >> 2, total = rows * d4;
  for (int t0 = threadIdx.x; t0 < total; t0 += ATT_THREADS * U) {
    float4 f[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const int t = t0 + u * ATT_THREADS;
      f[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (t < total) {
        const int r = t / d4, d = (t - r * d4) * 4, tok = row0 + r;
        if (tok < N) f[u] = *reinterpret_cast<const float4*>(src + (((size_t)b * N + tok) * nh + h) * dim + d);
      }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      const int t = t0 + u * ATT_THREADS;
      if (t < total) {
        const int r = t / d4, d = (t - r * d4) * 4;
        float* o = dst + r * ld + d;  // ld may be odd (kd + 1): scalar stores
        o[0] = f[u].x; o[1] = f[u].y; o[2] = f[u].z; o[3] = f[u].w;
      }
    }
  }
}

__global__ void __launch_bounds__(ATT_THREADS) attn_forward_tiled(const float* __restrict__ q, const float* __restrict__ k,
                                                                  const float* __restrict__ v, float* __restrict__ out,
                                                                  float* __restrict__ row_max, float* __restrict__ row_sum, int N,
                                                                  int nh, int kd, int hd, float scale) {
  extern __shared__ float sm[];
  const int ldk = kd + 1, ldv = hd + 1;
  float* Ks = sm;                  // [N][kd + 1]
  float* Vs = Ks + (size_t)N * ldk;  // [N][hd + 1]
  float* Qs = Vs + (size_t)N * ldv;  // [AT_T][kd]
  float* Ps = Qs + AT_T * kd;      // [AT_T][N]
  const int i0 = blockIdx.x * AT_T, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  load_head(Ks, k, b, h, N, nh, kd, ldk, 0, N);
  load_head(Vs, v, b, h, N, nh, hd, ldv, 0, N);
  load_head(Qs, q, b, h, N, nh, kd, kd, i0, AT_T);
  __syncthreads();
  const int r0 = warp * 2, r1 = r0 + 1;
  float* p0 = Ps + (size_t)r0 * N;
  float* p1 = Ps + (size_t)r1 * N;
  float m0 = -INFINITY, m1 = -INFINITY;
  for (int j = lane; j < N; j += 32) {
    float s0 = 0.f, s1 = 0.f;
    for (int d = 0; d < kd; d++) {
      const float kv = Ks[j * ldk + d];
      s0 = fmaf(Qs[r0 * kd + d], kv, s0);
      s1 = fmaf(Qs[r1 * kd + d], kv, s1);
    }
    s0 *= scale; s1 *= scale;
    p0[j] = s0; p1[j] = s1;
    m0 = fmaxf(m0, s0); m1 = fmaxf(m1, s1);
  }
  m0 = warp_max(m0); m1 = warp_max(m1);
  float l0 = 0.f, l1 = 0.f;
  for (int j = lane; j < N; j += 32) {
    const float e0 = expf(p0[j] - m0), e1 = expf(p1[j] - m1);
    p0[j] = e0; p1[j] = e1;
    l0 += e0; l1 += e1;
  }
  l0 = warp_sum(l0); l1 = warp_sum(l1);
  __syncwarp();
  const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
  for (int d = lane; d < hd; d += 32) {
    float o0 = 0.f, o1 = 0.f;
    for (int j = 0; j < N; j++) {
      const float vv = Vs[j * ldv + d];
      o0 = fmaf(p0[j], vv, o0);
      o1 = fmaf(p1[j], vv, o1);
    }
    if (i0 + r0 < N) out[(((size_t)b * N + i0 + r0) * nh + h) * hd + d] = o0 * inv0;
    if (i0 + r1 < N) out[(((size_t)b * N + i0 + r1) * nh + h) * hd + d] = o1 * inv1;
  }
  if (lane == 0 && row_max) {
    if (i0 + r0 < N) { row_max[((size_t)b * nh + h) * N + i0 + r0] = m0; row_sum[((size_t)b * nh + h) * N + i0 + r0] = l0; }
    if (i0 + r1 < N) { row_max[((size_t)b * nh + h) * N + i0 + r1] = m1; row_sum[((size_t)b * nh + h) * N + i0 + r1] = l1; }
  }
}

// per query tile: D_i = sum_j p_ij dP_ij, dS_ij = p_ij (dP_ij - D_i), dQ_i = scale sum_j dS_ij k_j
__global__ void __launch_bounds__(ATT_THREADS) attn_backward_q_tiled(const float* __restrict__ q, const float* __restrict__ k,
                                                                     const float* __restrict__ v, const float* __restrict__ dout,
                                                                     const float* __restrict__ row_max, const float* __restrict__ row_sum,
                                                                     float* __restrict__ row_d, float* __restrict__ dq, int N, int nh,
                                                                     int kd, int hd, float scale) {
  extern __shared__ float sm[];
  const int ldk = kd + 1, ldv = hd + 1;
  float* Ks = sm;
  float* Vs = Ks + (size_t)N * ldk;
  float* Qs = Vs + (size_t)N * ldv;  // [AT_T][kd]
  float* Os = Qs + AT_T * kd;        // [AT_T][hd] dO rows
  float* Ps = Os + AT_T * hd;        // [AT_T][N]
  const int i0 = blockIdx.x * AT_T, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  load_head(Ks, k, b, h, N, nh, kd, ldk, 0, N);
  load_head(Vs, v, b, h, N, nh, hd, ldv, 0, N);
  load_head(Qs, q, b, h, N, nh, kd, kd, i0, AT_T);
  load_head(Os, dout, b, h, N, nh, hd, hd, i0, AT_T);
  __syncthreads();
  for (int rr = 0; rr < 2; rr++) {
    const int r = warp * 2 + rr, i = i0 + r;
    if (i >= N) continue;  // warp-uniform
    const size_t st = ((size_t)b * nh + h) * N + i;
    const float mx = row_max[st], inv = 1.0f / row_sum[st];
    float* pr = Ps + (size_t)r * N;
    float dsum = 0.f;
    for (int j = lane; j < N; j += 32) {
      float s = 0.f, dp = 0.f;
      for (int d = 0; d < kd; d++) s = fmaf(Qs[r * kd + d], Ks[j * ldk + d], s);
      for (int d = 0; d < hd; d++) dp = fmaf(Os[r * hd + d], Vs[j * ldv + d], dp);
      const float pj = expf(s * scale - mx) * inv;
      pr[j] = pj;
      dsum = fmaf(pj, dp, dsum);
    }
    const float D = warp_sum(dsum);
    for (int j = lane; j < N; j += 32) {
      float dp = 0.f;
      for (int d = 0; d < hd; d++) dp = fmaf(Os[r * hd + d], Vs[j * ldv + d], dp);
      pr[j] = pr[j] * (dp - D);
    }
    __syncwarp();
    for (int d = lane; d < kd; d += 32) {
      float a = 0.f;
      for (int j = 0; j < N; j++) a = fmaf(pr[j], Ks[j * ldk + d], a);
      dq[(((size_t)b * N + i) * nh + h) * kd + d] = a * scale;
    }
    if (lane == 0) row_d[st] = D;
  }
}

// per key tile: dV_j = sum_i p_ij dO_i, dK_j = scale sum_i dS_ij q_i
__global__ void __launch_bounds__(ATT_THREADS) attn_backward_kv_tiled(const float* __restrict__ q, const float* __restrict__ k,
                                                                      const float* __restrict__ v, const float* __restrict__ dout,
                                                                      const float* __restrict__ row_max, const float* __restrict__ row_sum,
                                                                      const float* __restrict__ row_d, float* __restrict__ dk,
                                                                      float* __restrict__ dv, int N, int nh, int kd, int hd, float scale) {
  extern __shared__ float sm[];
  const int ldk = kd + 1, ldv = hd + 1;
  float* Qs = sm;                       // [N][kd + 1] all queries of the head
  float* Os = Qs + (size_t)N * ldk;     // [N][hd + 1] all dO rows
  float* St = Os + (size_t)N * ldv;     // [3][N] row max | 1 / row sum | D
  float* Kt = St + 3 * (size_t)N;       // [AT_T][kd]
  float* Vt = Kt + AT_T * kd;           // [AT_T][hd]
  float* Ps = Vt + AT_T * hd;           // [AT_T][N]
  const int j0 = blockIdx.x * AT_T, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  load_head(Qs, q, b, h, N, nh, kd, ldk, 0, N);
  load_head(Os, dout, b, h, N, nh, hd, ldv, 0, N);
  load_head(Kt, k, b, h, N, nh, kd, kd, j0, AT_T);
  load_head(Vt, v, b, h, N, nh, hd, hd, j0, AT_T);
  for (int i = threadIdx.x; i < N; i += ATT_THREADS) {
    const size_t st = ((size_t)b * nh + h) * N + i;
    St[i] = row_max[st];
    St[N + i] = 1.0f / row_sum[st];
    St[2 * N + i] = row_d[st];
  }
  __syncthreads();
  for (int rr = 0; rr < 2; rr++) {
    const int r = warp * 2 + rr, j = j0 + r;
    if (j >= N) continue;  // warp-uniform
    float* pr = Ps + (size_t)r * N;
    for (int i = lane; i < N; i += 32) {
      float s = 0.f;
      for (int d = 0; d < kd; d++) s = fmaf(Qs[i * ldk + d], Kt[r * kd + d], s);
      pr[i] = expf(s * scale - St[i]) * St[N + i];
    }
    __syncwarp();
    for (int d = lane; d < hd; d += 32) {
      float a = 0.f;
      for (int i = 0; i < N; i++) a = fmaf(pr[i], Os[i * ldv + d], a);
      dv[(((size_t)b * N + j) * nh + h) * hd + d] = a;
    }
    __syncwarp();
    for (int i = lane; i < N; i += 32) {
      float dp = 0.f;
      for (int d = 0; d < hd; d++) dp = fmaf(Os[i * ldv + d], Vt[r * hd + d], dp);
      pr[i] = pr[i] * (dp - St[2 * N + i]);
    }
    __syncwarp();
    for (int d = lane; d < kd; d += 32) {
      float a = 0.f;
      for (int i = 0; i < N; i++) a = fmaf(pr[i], Qs[i * ldk + d], a);
      dk[(((size_t)b * N + j) * nh + h) * kd + d] = a * scale;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Register-blocked backward for kd = 32, hd = 64 (every YOLOv11 size), same blocking as the forward kernel
// (kernels_generic.cu::attention_tiled_32x64_kernel): 16-byte shared-memory reads, two rows per warp sharing every
// operand, global fills as batches of independent vector loads.  Row strides 36 (K / Q) and 68 (V / dO) floats keep
// both "a lane owns a row" (LDS.128 along the row) and "a lane owns a channel" (scalar / LDS.64 down a column) reads
// bank-conflict free.  D_i = sum_d dO_id O_id (= sum_j P_ij dP_ij) comes from the recomputed forward output.
// ---------------------------------------------------------------------------------------------------------------
constexpr int AB_T = 16, AB_THREADS = 256, AB_LDK = 36, AB_LDV = 68;
__device__ __forceinline__ float4 lds4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float dot4(const float4& a, const float4& b, float acc) {
  acc = fmaf(a.x, b.x, acc); acc = fmaf(a.y, b.y, acc); acc = fmaf(a.z, b.z, acc); return fmaf(a.w, b.w, acc);
}
// rows [row0, row0 + rows) of one head of a (B, N, nh, dim) tensor -> smem with row stride ld (multiple of 4); rows >= N zero
template <int DIM>
__device__ __forceinline__ void fill_head(float* dst, int ld, const float* src, int b, int h, int N, int nh, int row0, int rows) {
  constexpr int U = 8, D4 = DIM / 4;
  const int total = rows * D4;
  for (int t0 = threadIdx.x; t0 < total; t0 += AB_THREADS * U) {
    float4 f[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const int t = t0 + u * AB_THREADS;
      f[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (t < total) {
        const int r = t / D4, d = (t - r * D4) * 4, tok = row0 + r;
        if (tok < N) f[u] = *reinterpret_cast<const float4*>(src + (((size_t)b * N + tok) * nh + h) * DIM + d);
      }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      const int t = t0 + u * AB_THREADS;
      if (t < total) {
        const int r = t / D4, d = (t - r * D4) * 4;
        *reinterpret_cast<float4*>(dst + (size_t)r * ld + d) = f[u];
      }
    }
  }
}

__global__ void __launch_bounds__(AB_THREADS, 1) attn_bwd_q_32x64(const float* __restrict__ q, const float* __restrict__ k,
                                                                 const float* __restrict__ v, const float* __restrict__ dout,
                                                                 const float* __restrict__ o, const float* __restrict__ row_max,
                                                                 const float* __restrict__ row_sum, float* __restrict__ row_d,
                                                                 float* __restrict__ dq, int N, int nh, float scale) {
  extern __shared__ __align__(16) float sm[];
  const int NK = (N + 31) & ~31, NP = (N + 3) & ~3;
  float* Ks = sm;                          // [NK][36]
  float* Vs = Ks + (size_t)NK * AB_LDK;    // [NK][68]
  float* Qs = Vs + (size_t)NK * AB_LDV;    // [16][32]
  float* Os = Qs + AB_T * 32;              // [16][64] dO rows
  float* Ps = Os + AB_T * 64;              // [16][NP] dS
  const int i0 = blockIdx.x * AB_T, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  fill_head<32>(Ks, AB_LDK, k, b, h, N, nh, 0, NK);
  fill_head<64>(Vs, AB_LDV, v, b, h, N, nh, 0, NK);
  fill_head<32>(Qs, 32, q, b, h, N, nh, i0, AB_T);
  fill_head<64>(Os, 64, dout, b, h, N, nh, i0, AB_T);
  __syncthreads();
  const int r0 = warp * 2, r1 = r0 + 1;
  const bool ok0 = i0 + r0 < N, ok1 = i0 + r1 < N;
  // D = dO . O per row (two channels per lane)
  float D0 = 0.f, D1 = 0.f;
  {
    const size_t base0 = (((size_t)b * N + min(i0 + r0, N - 1)) * nh + h) * 64 + 2 * lane;
    const size_t base1 = (((size_t)b * N + min(i0 + r1, N - 1)) * nh + h) * 64 + 2 * lane;
    const float2 o0 = *reinterpret_cast<const float2*>(o + base0), o1 = *reinterpret_cast<const float2*>(o + base1);
    D0 = Os[r0 * 64 + 2 * lane] * o0.x + Os[r0 * 64 + 2 * lane + 1] * o0.y;
    D1 = Os[r1 * 64 + 2 * lane] * o1.x + Os[r1 * 64 + 2 * lane + 1] * o1.y;
    for (int s = 16; s; s >>= 1) { D0 += __shfl_xor_sync(0xffffffffu, D0, s); D1 += __shfl_xor_sync(0xffffffffu, D1, s); }
  }
  const size_t st0 = ((size_t)b * nh + h) * N + min(i0 + r0, N - 1), st1 = ((size_t)b * nh + h) * N + min(i0 + r1, N - 1);
  const float mx0 = row_max[st0], inv0 = 1.0f / row_sum[st0], mx1 = row_max[st1], inv1 = 1.0f / row_sum[st1];
  float q0[32], q1[32];
#pragma unroll
  for (int d = 0; d < 32; d += 4) {
    const float4 a = lds4(Qs + r0 * 32 + d), c = lds4(Qs + r1 * 32 + d);
    q0[d] = a.x; q0[d + 1] = a.y; q0[d + 2] = a.z; q0[d + 3] = a.w;
    q1[d] = c.x; q1[d + 1] = c.y; q1[d + 2] = c.z; q1[d + 3] = c.w;
  }
  float* p0 = Ps + (size_t)r0 * NP;
  float* p1 = Ps + (size_t)r1 * NP;
  for (int j = lane; j < NK; j += 32) {
    const float* kr = Ks + (size_t)j * AB_LDK;
    const float* vr = Vs + (size_t)j * AB_LDV;
    float s0 = 0.f, s1 = 0.f, dp0 = 0.f, dp1 = 0.f;
#pragma unroll
    for (int d = 0; d < 32; d += 4) {
      const float4 kv = lds4(kr + d);
      s0 = fmaf(q0[d], kv.x, s0); s1 = fmaf(q1[d], kv.x, s1);
      s0 = fmaf(q0[d + 1], kv.y, s0); s1 = fmaf(q1[d + 1], kv.y, s1);
      s0 = fmaf(q0[d + 2], kv.z, s0); s1 = fmaf(q1[d + 2], kv.z, s1);
      s0 = fmaf(q0[d + 3], kv.w, s0); s1 = fmaf(q1[d + 3], kv.w, s1);
    }
#pragma unroll
    for (int d = 0; d < 64; d += 4) {
      const float4 vv = lds4(vr + d);
      dp0 = dot4(lds4(Os + r0 * 64 + d), vv, dp0);
      dp1 = dot4(lds4(Os + r1 * 64 + d), vv, dp1);
    }
    if (j < NP) {
      const bool in = j < N;
      p0[j] = in ? expf(s0 * scale - mx0) * inv0 * (dp0 - D0) : 0.f;
      p1[j] = in ? expf(s1 * scale - mx1) * inv1 * (dp1 - D1) : 0.f;
    }
  }
  __syncwarp();
  float a0 = 0.f, a1 = 0.f;
  for (int j = 0; j < NP; j += 4) {
    const float4 da = lds4(p0 + j), db = lds4(p1 + j);
    const float k0 = Ks[(size_t)j * AB_LDK + lane], k1 = Ks[(size_t)(j + 1) * AB_LDK + lane];
    const float k2 = Ks[(size_t)(j + 2) * AB_LDK + lane], k3 = Ks[(size_t)(j + 3) * AB_LDK + lane];
    a0 = fmaf(da.x, k0, a0); a1 = fmaf(db.x, k0, a1);
    a0 = fmaf(da.y, k1, a0); a1 = fmaf(db.y, k1, a1);
    a0 = fmaf(da.z, k2, a0); a1 = fmaf(db.z, k2, a1);
    a0 = fmaf(da.w, k3, a0); a1 = fmaf(db.w, k3, a1);
  }
  if (ok0) dq[(((size_t)b * N + i0 + r0) * nh + h) * 32 + lane] = a0 * scale;
  if (ok1) dq[(((size_t)b * N + i0 + r1) * nh + h) * 32 + lane] = a1 * scale;
  if (lane == 0) {
    if (ok0) row_d[st0] = D0;
    if (ok1) row_d[st1] = D1;
  }
}

__global__ void __launch_bounds__(AB_THREADS, 1) attn_bwd_kv_32x64(const float* __restrict__ q, const float* __restrict__ k,
                                                                  const float* __restrict__ v, const float* __restrict__ dout,
                                                                  const float* __restrict__ row_max, const float* __restrict__ row_sum,
                                                                  const float* __restrict__ row_d, float* __restrict__ dk,
                                                                  float* __restrict__ dv, int N, int nh, float scale) {
  extern __shared__ __align__(16) float sm[];
  const int NK = (N + 31) & ~31, NP = (N + 3) & ~3;
  float* Qs = sm;                          // [NK][36] all queries of the head
  float* Os = Qs + (size_t)NK * AB_LDK;    // [NK][68] all dO rows
  float* St = Os + (size_t)NK * AB_LDV;    // [3][NK] row max | 1 / row sum | D
  float* Kt = St + 3 * (size_t)NK;         // [16][32]
  float* Vt = Kt + AB_T * 32;              // [16][64]
  float* Ps = Vt + AB_T * 64;              // [16][NP]
  const int j0 = blockIdx.x * AB_T, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  fill_head<32>(Qs, AB_LDK, q, b, h, N, nh, 0, NK);
  fill_head<64>(Os, AB_LDV, dout, b, h, N, nh, 0, NK);
  fill_head<32>(Kt, 32, k, b, h, N, nh, j0, AB_T);
  fill_head<64>(Vt, 64, v, b, h, N, nh, j0, AB_T);
  for (int i = threadIdx.x; i < NK; i += AB_THREADS) {
    const size_t st = ((size_t)b * nh + h) * N + min(i, N - 1);
    St[i] = row_max[st];
    St[NK + i] = i < N ? 1.0f / row_sum[st] : 0.f;  // padded queries get p = 0
    St[2 * NK + i] = row_d[st];
  }
  __syncthreads();
  const int r0 = warp * 2, r1 = r0 + 1;
  const bool ok0 = j0 + r0 < N, ok1 = j0 + r1 < N;
  float k0[32], k1[32];
#pragma unroll
  for (int d = 0; d < 32; d += 4) {
    const float4 a = lds4(Kt + r0 * 32 + d), c = lds4(Kt + r1 * 32 + d);
    k0[d] = a.x; k0[d + 1] = a.y; k0[d + 2] = a.z; k0[d + 3] = a.w;
    k1[d] = c.x; k1[d + 1] = c.y; k1[d + 2] = c.z; k1[d + 3] = c.w;
  }
  float* p0 = Ps + (size_t)r0 * NP;
  float* p1 = Ps + (size_t)r1 * NP;
  // P^T rows of the two keys
  for (int i = lane; i < NK; i += 32) {
    const float* qr = Qs + (size_t)i * AB_LDK;
    float s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int d = 0; d < 32; d += 4) {
      const float4 qv = lds4(qr + d);
      s0 = fmaf(qv.x, k0[d], s0); s1 = fmaf(qv.x, k1[d], s1);
      s0 = fmaf(qv.y, k0[d + 1], s0); s1 = fmaf(qv.y, k1[d + 1], s1);
      s0 = fmaf(qv.z, k0[d + 2], s0); s1 = fmaf(qv.z, k1[d + 2], s1);
      s0 = fmaf(qv.w, k0[d + 3], s0); s1 = fmaf(qv.w, k1[d + 3], s1);
    }
    if (i < NP) {
      p0[i] = expf(s0 * scale - St[i]) * St[NK + i];
      p1[i] = expf(s1 * scale - St[i]) * St[NK + i];
    }
  }
  __syncwarp();
  {  // dV_j = sum_i p_ij dO_i: a lane owns channels 2 lane, 2 lane + 1
    float a00 = 0.f, a01 = 0.f, a10 = 0.f, a11 = 0.f;
    const float* ocol = Os + 2 * lane;
    for (int i = 0; i < NP; i += 4) {
      const float4 pa = lds4(p0 + i), pb = lds4(p1 + i);
      const float2 o0 = *reinterpret_cast<const float2*>(ocol + (size_t)i * AB_LDV);
      const float2 o1 = *reinterpret_cast<const float2*>(ocol + (size_t)(i + 1) * AB_LDV);
      const float2 o2 = *reinterpret_cast<const float2*>(ocol + (size_t)(i + 2) * AB_LDV);
      const float2 o3 = *reinterpret_cast<const float2*>(ocol + (size_t)(i + 3) * AB_LDV);
      a00 = fmaf(pa.x, o0.x, a00); a01 = fmaf(pa.x, o0.y, a01); a10 = fmaf(pb.x, o0.x, a10); a11 = fmaf(pb.x, o0.y, a11);
      a00 = fmaf(pa.y, o1.x, a00); a01 = fmaf(pa.y, o1.y, a01); a10 = fmaf(pb.y, o1.x, a10); a11 = fmaf(pb.y, o1.y, a11);
      a00 = fmaf(pa.z, o2.x, a00); a01 = fmaf(pa.z, o2.y, a01); a10 = fmaf(pb.z, o2.x, a10); a11 = fmaf(pb.z, o2.y, a11);
      a00 = fmaf(pa.w, o3.x, a00); a01 = fmaf(pa.w, o3.y, a01); a10 = fmaf(pb.w, o3.x, a10); a11 = fmaf(pb.w, o3.y, a11);
    }
    if (ok0) *reinterpret_cast<float2*>(dv + (((size_t)b * N + j0 + r0) * nh + h) * 64 + 2 * lane) = make_float2(a00, a01);
    if (ok1) *reinterpret_cast<float2*>(dv + (((size_t)b * N + j0 + r1) * nh + h) * 64 + 2 * lane) = make_float2(a10, a11);
  }
  __syncwarp();
  // dS^T = P^T o (dP^T - D): dP_ij = dO_i . v_j, v rows broadcast from the tile
  for (int i = lane; i < NK; i += 32) {
    const float* orow = Os + (size_t)i * AB_LDV;
    float dp0 = 0.f, dp1 = 0.f;
#pragma unroll
    for (int d = 0; d < 64; d += 4) {
      const float4 ov = lds4(orow + d);
      dp0 = dot4(ov, lds4(Vt + r0 * 64 + d), dp0);
      dp1 = dot4(ov, lds4(Vt + r1 * 64 + d), dp1);
    }
    if (i < NP) {
      p0[i] = p0[i] * (dp0 - St[2 * NK + i]);
      p1[i] = p1[i] * (dp1 - St[2 * NK + i]);
    }
  }
  __syncwarp();
  float a0 = 0.f, a1 = 0.f;  // dK_j = scale sum_i dS_ij q_i: a lane owns channel `lane`
  for (int i = 0; i < NP; i += 4) {
    const float4 da = lds4(p0 + i), db = lds4(p1 + i);
    const float q0v = Qs[(size_t)i * AB_LDK + lane], q1v = Qs[(size_t)(i + 1) * AB_LDK + lane];
    const float q2v = Qs[(size_t)(i + 2) * AB_LDK + lane], q3v = Qs[(size_t)(i + 3) * AB_LDK + lane];
    a0 = fmaf(da.x, q0v, a0); a1 = fmaf(db.x, q0v, a1);
    a0 = fmaf(da.y, q1v, a0); a1 = fmaf(db.y, q1v, a1);
    a0 = fmaf(da.z, q2v, a0); a1 = fmaf(db.z, q2v, a1);
    a0 = fmaf(da.w, q3v, a0); a1 = fmaf(db.w, q3v, a1);
  }
  if (ok0) dk[(((size_t)b * N + j0 + r0) * nh + h) * 32 + lane] = a0 * scale;
  if (ok1) dk[(((size_t)b * N + j0 + r1) * nh + h) * 32 + lane] = a1 * scale;
}

static size_t ab_smem_bytes(int N, int which) {  // which: 0 q pass, 1 kv pass
  const size_t NK = (N + 31) & ~31, NP = (N + 3) & ~3;
  const size_t heads = NK * AB_LDK + NK * AB_LDV;
  return (heads + (which ? 3 * NK : 0) + (size_t)AB_T * (32 + 64) + (size_t)AB_T * NP) * sizeof(float);
}
static bool ab_fits(int N) { return ab_smem_bytes(N, 1) <= 227 * 1024 && ab_smem_bytes(N, 0) <= 227 * 1024; }

static size_t attn_tiled_smem(int N, int kd, int hd, int which) {  // floats; which: 0 forward, 1 backward q, 2 backward kv
  const size_t heads = (size_t)N * (kd + 1) + (size_t)N * (hd + 1);
  if (which == 0) return heads + (size_t)AT_T * kd + (size_t)AT_T * N;
  if (which == 1) return heads + (size_t)AT_T * (kd + hd) + (size_t)AT_T * N;
  return heads + 3 * (size_t)N + (size_t)AT_T * (kd + hd) + (size_t)AT_T * N;
}
static bool attn_tiled_ok(int N, int kd, int hd) { return attn_tiled_smem(N, kd, hd, 2) * sizeof(float) <= 200 * 1024; }

static int attn_check(int B, int N, int nh, int kd, int hd, size_t smem_floats) {
  if (B <= 0 || N <= 0 || nh <= 0 || kd <= 0 || hd <= 0) { set_error("attention: bad shape"); return YB_ERR_SHAPE; }
  if (smem_floats * sizeof(float) > 200 * 1024) { set_error("attention: N too large for the shared-memory score rows"); return YB_ERR_NOT_IMPLEMENTED; }
  return 0;
}

int attention_forward_f32(const float* q, const float* k, const float* v, int B, int N, int nh, int kd, int hd, float scale,
                          float* out, float* row_max, float* row_sum, cudaStream_t s) {
  const size_t smem = (size_t)N + kd;
  if (int rc = attn_check(B, N, nh, kd, hd, smem)) return rc;
  if (kd == 32 && hd == 64 && attention_tiled_32x64_fits(N)) {  // register-blocked kernel shared with the inference engine
    AttnIO io;
    io.q = q; io.k = k; io.v = v;
    io.in_tok = (long long)nh * kd; io.in_img = (long long)N * nh * kd;
    io.v_tok = (long long)nh * hd; io.v_img = (long long)N * nh * hd;
    io.q_head = io.k_head = kd; io.v_head = hd;
    io.out = out; io.out_tok = (long long)nh * hd; io.out_img = (long long)N * nh * hd;
    io.vout = nullptr; io.row_max = row_max; io.row_sum = row_sum;
    return launch_attention_tiled_32x64<float>(io, B, N, nh, scale, s);
  }
  if (attn_tiled_ok(N, kd, hd)) {
    YB_CUDA_CHECK(cudaFuncSetAttribute(attn_forward_tiled, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attn_forward_tiled<<<dim3((N + AT_T - 1) / AT_T, nh, B), ATT_THREADS, attn_tiled_smem(N, kd, hd, 0) * sizeof(float), s>>>(
        q, k, v, out, row_max, row_sum, N, nh, kd, hd, scale);
    YB_CUDA_CHECK(cudaGetLastError());
    return 0;
  }
  YB_CUDA_CHECK(cudaFuncSetAttribute(attn_forward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  attn_forward_kernel<<<dim3(N, nh, B), AT_THREADS, smem * sizeof(float), s>>>(q, k, v, out, row_max, row_sum, N, nh, kd, hd, scale);
  YB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int attention_backward_f32(const float* q, const float* k, const float* v, const float* dout, int B, int N, int nh, int kd,
                           int hd, float scale, float* dq, float* dk, float* dv, cudaStream_t s) {
  const size_t smem_q = (size_t)N + kd + hd, smem_kv = (size_t)2 * N + kd + hd;
  if (int rc = attn_check(B, N, nh, kd, hd, smem_kv)) return rc;
  float* stats = nullptr;  // row max | row sum | row D, each (B, nh, N)
  const size_t n = (size_t)B * nh * N;
  YB_CUDA_CHECK(cudaMallocAsync((void**)&stats, (3 * n + (size_t)B * N * nh * hd) * sizeof(float), s));
  float* tmp_out = stats + 3 * n;  // the forward output is recomputed only for its row statistics
  int rc = attention_forward_f32(q, k, v, B, N, nh, kd, hd, scale, tmp_out, stats, stats + n, s);
  if (!rc && kd == 32 && hd == 64 && ab_fits(N)) {
    cudaFuncSetAttribute(attn_bwd_q_32x64, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaFuncSetAttribute(attn_bwd_kv_32x64, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    const dim3 grid((N + AB_T - 1) / AB_T, nh, B);
    attn_bwd_q_32x64<<<grid, AB_THREADS, ab_smem_bytes(N, 0), s>>>(q, k, v, dout, tmp_out, stats, stats + n, stats + 2 * n, dq, N, nh, scale);
    attn_bwd_kv_32x64<<<grid, AB_THREADS, ab_smem_bytes(N, 1), s>>>(q, k, v, dout, stats, stats + n, stats + 2 * n, dk, dv, N, nh, scale);
    if (cudaGetLastError() != cudaSuccess) { set_error("attention backward launch failed"); rc = YB_ERR_CUDA; }
  } else if (!rc && attn_tiled_ok(N, kd, hd)) {
    cudaFuncSetAttribute(attn_backward_q_tiled, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(attn_backward_kv_tiled, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    const dim3 grid((N + AT_T - 1) / AT_T, nh, B);
    attn_backward_q_tiled<<<grid, ATT_THREADS, attn_tiled_smem(N, kd, hd, 1) * sizeof(float), s>>>(q, k, v, dout, stats, stats + n,
                                                                                                   stats + 2 * n, dq, N, nh, kd, hd, scale);
    attn_backward_kv_tiled<<<grid, ATT_THREADS, attn_tiled_smem(N, kd, hd, 2) * sizeof(float), s>>>(q, k, v, dout, stats, stats + n,
                                                                                                    stats + 2 * n, dk, dv, N, nh, kd, hd, scale);
    if (cudaGetLastError() != cudaSuccess) { set_error("attention backward launch failed"); rc = YB_ERR_CUDA; }
  } else if (!rc) {
    cudaFuncSetAttribute(attn_backward_q_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(attn_backward_kv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    attn_backward_q_kernel<<<dim3(N, nh, B), AT_THREADS, smem_q * sizeof(float), s>>>(q, k, v, dout, stats, stats + n, stats + 2 * n,
                                                                                      dq, N, nh, kd, hd, scale);
    attn_backward_kv_kernel<<<dim3(N, nh, B), AT_THREADS, smem_kv * sizeof(float), s>>>(q, k, v, dout, stats, stats + n, stats + 2 * n,
                                                                                        dk, dv, N, nh, kd, hd, scale);
    if (cudaGetLastError() != cudaSuccess) { set_error("attention backward launch failed"); rc = YB_ERR_CUDA; }
  }
  cudaFreeAsync(stats, s);
  return rc;
}

}  // namespace yb

using namespace yb;

static bool have_dev(const char* who) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    set_error(std::string(who) + ": no CUDA device");
    return false;
  }
  return true;
}

extern "C" {

int32_t yb_dwconv3x3_forward_f32(const float* x, const float* w, int32_t n, int32_t height, int32_t width, int32_t channels,
                                 float* z, void* stream) {
  if (!x || !w || !z || n <= 0 || height <= 0 || width <= 0 || channels <= 0) { set_error("yb_dwconv3x3_forward_f32: bad argument"); return YB_ERR_INVALID_ARG; }
  if (!have_dev("yb_dwconv3x3_forward_f32")) return YB_ERR_NO_DEVICE;
  return dwconv3x3_forward_f32(x, w, n, height, width, channels, z, (cudaStream_t)stream);
}

int32_t yb_dwconv3x3_backward_f32(const float* x, const float* dz, const float* w, int32_t n, int32_t height, int32_t width,
                                  int32_t channels, float* dx, float* dw, void* stream) {
  if (!x || !dz || !w || !dx || !dw || n <= 0 || height <= 0 || width <= 0 || channels <= 0) { set_error("yb_dwconv3x3_backward_f32: bad argument"); return YB_ERR_INVALID_ARG; }
  if (!have_dev("yb_dwconv3x3_backward_f32")) return YB_ERR_NO_DEVICE;
  return dwconv3x3_backward_f32(x, dz, w, n, height, width, channels, dx, dw, (cudaStream_t)stream);
}

int32_t yb_attention_forward_f32(const float* q, const float* k, const float* v, int32_t batch, int32_t tokens, int32_t heads,
                                 int32_t key_dim, int32_t head_dim, float scale, float* out, void* stream) {
  if (!q || !k || !v || !out) { set_error("yb_attention_forward_f32: null argument"); return YB_ERR_INVALID_ARG; }
  if (!have_dev("yb_attention_forward_f32")) return YB_ERR_NO_DEVICE;
  return attention_forward_f32(q, k, v, batch, tokens, heads, key_dim, head_dim, scale, out, nullptr, nullptr, (cudaStream_t)stream);
}

int32_t yb_attention_backward_f32(const float* q, const float* k, const float* v, const float* dout, int32_t batch, int32_t tokens,
                                  int32_t heads, int32_t key_dim, int32_t head_dim, float scale, float* dq, float* dk, float* dv,
                                  void* stream) {
  if (!q || !k || !v || !dout || !dq || !dk || !dv) { set_error("yb_attention_backward_f32: null argument"); return YB_ERR_INVALID_ARG; }
  if (!have_dev("yb_attention_backward_f32")) return YB_ERR_NO_DEVICE;
  return attention_backward_f32(q, k, v, dout, batch, tokens, heads, key_dim, head_dim, scale, dq, dk, dv, (cudaStream_t)stream);
}

}  // extern "C"
