// CUDA-core kernels of the yolob200 engine, templated on the activation storage type.
//   T = float  : parity mode (fp32 storage, fp32 FMA) - matches the fp32 oracle to ~1e-5
//   T = __half : debug twin of the tensor-core path (same fp16 storage/weights, fp32 accumulate)
// plus the HBM-bound glue ops used by both modes (SPPF pool, upsample, decode, layout).
// Reference ops restated: Modules/Convs.cs:36-56 (Conv), Block.cs:236-282 (SPPF),
// Head.cs:204-223 + Block.cs:15-45 + Utils/Tal.cs:313-356 (decode).
#include <algorithm>

#include "common.cuh"

namespace yb {

// ------------------------------------------------------------------------------------------
// Generic implicit-GEMM convolution on CUDA cores.
//   M = B*Ho*Wo output pixels, N = Cout, K = k*k*Cin (tap-major).  64x64 tile, 16-deep slabs,
//   256 threads x (4 px x 4 cout) register tile.  Weights fp32 [tap][Cin][Cout].
// ------------------------------------------------------------------------------------------
constexpr int GT_M = 64, GT_N = 64, GT_K = 16;

template <typename T>
__global__ void __launch_bounds__(256) conv_generic_kernel(ConvParams p, int M) {
  __shared__ float As[GT_K][GT_M + 4];
  __shared__ __align__(16) float Bs[GT_K][GT_N];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.x * GT_M, n0 = blockIdx.y * GT_N;
  const float* __restrict__ w = reinterpret_cast<const float*>(p.w);
  const T* __restrict__ in = reinterpret_cast<const T*>(p.in.base);

  // A-load role: pixel (tid/4), channel quad (tid%4)*4
  const int a_px = tid >> 2, a_cq = (tid & 3) * 4;
  const int am = m0 + a_px;
  int an = 0, aho = 0, awo = 0;
  const bool a_valid = am < M;
  if (a_valid) {
    an = am / (p.Ho * p.Wo);
    int r = am - an * p.Ho * p.Wo;
    aho = r / p.Wo;
    awo = r - aho * p.Wo;
  }
  // B-load role: k row (tid/16), cout quad (tid%16)*4
  const int b_k = tid >> 4, b_c = (tid & 15) * 4;

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) acc[i][j] = 0.f;

  const int taps = p.k * p.k;
  for (int t = 0; t < taps; t++) {
    const int kh = t / p.k, kw = t - kh * p.k;
    const int hi = aho * p.stride + kh - p.pad;
    const int wi = awo * p.stride + kw - p.pad;
    const bool pix_ok = a_valid && hi >= 0 && hi < p.in.H && wi >= 0 && wi < p.in.W;
    const T* src = pix_ok ? in + ((size_t)(an * p.in.H + hi) * p.in.W + wi) * p.in.pitch + p.in.coff : in;
    for (int c0 = 0; c0 < p.Cin; c0 += GT_K) {
      float av[4];
#pragma unroll
      for (int q = 0; q < 4; q++) {
        const int c = c0 + a_cq + q;
        av[q] = (pix_ok && c < p.Cin) ? to_f<T>(src[c]) : 0.f;
      }
#pragma unroll
      for (int q = 0; q < 4; q++) As[a_cq + q][a_px] = av[q];
      {
        const int c = c0 + b_k;
        const float* wr = w + ((size_t)t * p.Cin + c) * p.Cout + n0 + b_c;
#pragma unroll
        for (int q = 0; q < 4; q++)
          Bs[b_k][b_c + q] = (c < p.Cin && n0 + b_c + q < p.Cout) ? wr[q] : 0.f;
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < GT_K; kk++) {
        float a[4], b[4];
#pragma unroll
        for (int i = 0; i < 4; i++) a[i] = As[kk][ty * 4 + i];
        const float4 bv = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
        b[0] = bv.x; b[1] = bv.y; b[2] = bv.z; b[3] = bv.w;
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
          for (int j = 0; j < 4; j++) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
      __syncthreads();
    }
  }

  T* __restrict__ out = reinterpret_cast<T*>(p.out.base);
  const T* __restrict__ res = reinterpret_cast<const T*>(p.res.base);
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
    const size_t opix = (size_t)m;  // output pixels are dense (n,ho,wo) in the out buffer
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int co = n0 + tx * 4 + j;
      if (co >= p.Cout) continue;
      float v = acc[i][j] + p.bias[co];
      if (p.act == ACT_SILU) v = silu_f(v);
      if (res) v += to_f<T>(res[opix * p.res.pitch + p.res.coff + co]);
      out[opix * p.out.pitch + p.out.coff + co] = from_f<T>(v);
    }
  }
}

template <typename T>
int launch_conv_generic(const ConvParams& p, cudaStream_t s) {
  const int M = p.B * p.Ho * p.Wo;
  dim3 grid((M + GT_M - 1) / GT_M, (p.Cout + GT_N - 1) / GT_N);
  conv_generic_kernel<T><<<grid, 256, 0, s>>>(p, M);
  YB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
template int launch_conv_generic<float>(const ConvParams&, cudaStream_t);
template int launch_conv_generic<__half>(const ConvParams&, cudaStream_t);

// ------------------------------------------------------------------------------------------
// Depthwise 3x3 stride-1 pad-1 conv + bias + act (Convs.cs:108-114 DWConv, Block.cs:746 pe).
// HBM-bound: one thread per (pixel, channel), channels fastest -> coalesced.
// ------------------------------------------------------------------------------------------
template <typename T>
__global__ void dwconv3x3_kernel(ConvParams p, size_t total) {
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c = idx % p.Cout;
  size_t pix = idx / p.Cout;
  const int wo = pix % p.Wo;
  const int ho = (pix / p.Wo) % p.Ho;
  const int n = pix / ((size_t)p.Wo * p.Ho);
  const T* in = reinterpret_cast<const T*>(p.in.base);
  const float* w = reinterpret_cast<const float*>(p.w);
  float acc = 0.f;
#pragma unroll
  for (int kh = 0; kh < 3; kh++) {
    const int hi = ho + kh - 1;
    if (hi < 0 || hi >= p.in.H) continue;
#pragma unroll
    for (int kw = 0; kw < 3; kw++) {
      const int wi = wo + kw - 1;
      if (wi < 0 || wi >= p.in.W) continue;
      acc = fmaf(to_f<T>(in[((size_t)(n * p.in.H + hi) * p.in.W + wi) * p.in.pitch + p.in.coff + c]),
                 w[(kh * 3 + kw) * p.Cout + c], acc);
    }
  }
  float v = acc + p.bias[c];
  if (p.act == ACT_SILU) v = silu_f(v);
  const T* res = reinterpret_cast<const T*>(p.res.base);
  if (res) v += to_f<T>(res[pix * p.res.pitch + p.res.coff + c]);
  reinterpret_cast<T*>(p.out.base)[pix * p.out.pitch + p.out.coff + c] = from_f<T>(v);
}

// fp16 path, channels in groups of 8 (one 16-byte vector): a thread produces DW_PIX adjacent output pixels of one row
// for 8 channels from a 3 x (DW_PIX + 2) window of 16-byte loads (4.5 loads per output instead of 9 scalar ones), the
// 72 weights of its channel group in registers.  Consecutive threads = consecutive channel groups: every load / store
// instruction of a warp covers whole contiguous pixel rows.  (The scalar kernel above issues 9 scalar loads per output.)
constexpr int DW_PIX = 4;
__global__ void __launch_bounds__(256) dwconv3x3_h8_kernel(ConvParams p, int groups8, int wtiles, int total) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int g = idx % groups8;
  int t = idx / groups8;
  const int wt = t % wtiles; t /= wtiles;
  const int ho = t % p.Ho;
  const int n = t / p.Ho;
  const int c = g * 8;
  const int wo0 = wt * DW_PIX;
  const __half* in = reinterpret_cast<const __half*>(p.in.base) + p.in.coff + c;
  const float* w = reinterpret_cast<const float*>(p.w);
  float acc[DW_PIX][8];
#pragma unroll
  for (int q = 0; q < DW_PIX; q++)
#pragma unroll
    for (int j = 0; j < 8; j++) acc[q][j] = 0.f;
#pragma unroll
  for (int kh = 0; kh < 3; kh++) {
    const int hi = ho + kh - 1;
    if (hi < 0 || hi >= p.in.H) continue;
    float wk[3][8];
#pragma unroll
    for (int kw = 0; kw < 3; kw++) {
      const float4 a = *reinterpret_cast<const float4*>(w + (kh * 3 + kw) * p.Cout + c);
      const float4 b = *reinterpret_cast<const float4*>(w + (kh * 3 + kw) * p.Cout + c + 4);
      wk[kw][0] = a.x; wk[kw][1] = a.y; wk[kw][2] = a.z; wk[kw][3] = a.w;
      wk[kw][4] = b.x; wk[kw][5] = b.y; wk[kw][6] = b.z; wk[kw][7] = b.w;
    }
    const __half* row = in + (size_t)(n * p.in.H + hi) * p.in.W * p.in.pitch;
#pragma unroll
    for (int col = 0; col < DW_PIX + 2; col++) {
      const int wi = wo0 + col - 1;
      if (wi < 0 || wi >= p.in.W) continue;
      const int4 v = *reinterpret_cast<const int4*>(row + (size_t)wi * p.in.pitch);
      const __half2* h = reinterpret_cast<const __half2*>(&v);
      float x[8];
#pragma unroll
      for (int j = 0; j < 4; j++) { const float2 f = __half22float2(h[j]); x[2 * j] = f.x; x[2 * j + 1] = f.y; }
#pragma unroll
      for (int kw = 0; kw < 3; kw++) {
        const int q = col - kw;  // output pixel this column feeds through tap kw
        if (q >= 0 && q < DW_PIX) {
#pragma unroll
          for (int j = 0; j < 8; j++) acc[q][j] = fmaf(x[j], wk[kw][j], acc[q][j]);
        }
      }
    }
  }
  const float4 b0 = *reinterpret_cast<const float4*>(p.bias + c), b1 = *reinterpret_cast<const float4*>(p.bias + c + 4);
  const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
  const __half* res = reinterpret_cast<const __half*>(p.res.base);
#pragma unroll
  for (int q = 0; q < DW_PIX; q++) {
    const int wo = wo0 + q;
    if (wo >= p.Wo) break;
    const size_t pix = ((size_t)n * p.Ho + ho) * p.Wo + wo;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; j++) {
      v[j] = acc[q][j] + bb[j];
      if (p.act == ACT_SILU) v[j] = silu_f(v[j]);
    }
    if (res) {
      const int4 rv = *reinterpret_cast<const int4*>(res + pix * p.res.pitch + p.res.coff + c);
      const __half2* rh = reinterpret_cast<const __half2*>(&rv);
#pragma unroll
      for (int j = 0; j < 4; j++) { const float2 f = __half22float2(rh[j]); v[2 * j] += f.x; v[2 * j + 1] += f.y; }
    }
    int4 o;
    __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int j = 0; j < 4; j++) oh[j] = __floats2half2_rn(v[2 * j], v[2 * j + 1]);
    *reinterpret_cast<int4*>(reinterpret_cast<__half*>(p.out.base) + pix * p.out.pitch + p.out.coff + c) = o;
  }
}

template <typename T>
int launch_dwconv3x3(const ConvParams& p, cudaStream_t s) {
  const size_t total = (size_t)p.B * p.Ho * p.Wo * p.Cout;
  if (sizeof(T) == 2 && p.Cout % 8 == 0 && p.in.pitch % 8 == 0 && p.in.coff % 8 == 0 && p.out.pitch % 8 == 0 && p.out.coff % 8 == 0 &&
      (!p.res.base || (p.res.pitch % 8 == 0 && p.res.coff % 8 == 0)) && p.stride == 1 && p.Ho == p.in.H && p.Wo == p.in.W &&
      total / 8 < (size_t)1 << 30) {
    const int groups8 = p.Cout / 8, wtiles = (p.Wo + DW_PIX - 1) / DW_PIX;
    const int tot = p.B * p.Ho * wtiles * groups8;
    dwconv3x3_h8_kernel<<<(tot + 255) / 256, 256, 0, s>>>(p, groups8, wtiles, tot);
    YB_CUDA_CHECK(cudaGetLastError());
    return 0;
  }
  dwconv3x3_kernel<T><<<(unsigned)((total + 255) / 256), 256, 0, s>>>(p, total);
  YB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
template int launch_dwconv3x3<float>(const ConvParams&, cudaStream_t);
template int launch_dwconv3x3<__half>(const ConvParams&, cudaStream_t);

// ------------------------------------------------------------------------------------------
// SPPF pyramid (Block.cs:275-279): three cascaded MaxPool2d(5,1,2) of the cv1 output, written
// into concat slices 1..3.  One block = one image x 8 channels; the map lives in shared memory
// and each 5x5 pool is a row pass + column pass.  -inf padding like ATen's max_pool2d.
// ------------------------------------------------------------------------------------------
constexpr int SP_CC = 8;

template <typename T>
__global__ void __launch_bounds__(256) sppf_pool_kernel(View in, View o5, View o9, View o13) {
  extern __shared__ float sp_smem[];
  const int H = in.H, W = in.W;
  const int HW = H * W;
  float* a = sp_smem;
  float* b = a + HW * SP_CC;
  float* c = b + HW * SP_CC;
  const int n = blockIdx.y;
  const int c0 = blockIdx.x * SP_CC;
  const int cc = min(SP_CC, in.C - c0);
  const T* src = reinterpret_cast<const T*>(in.base);
  for (int i = threadIdx.x; i < HW * SP_CC; i += blockDim.x) {
    const int ch = i % SP_CC, pix = i / SP_CC;
    a[i] = ch < cc ? to_f<T>(src[((size_t)n * HW + pix) * in.pitch + in.coff + c0 + ch]) : 0.f;
  }
  __syncthreads();
  View outs[3] = {o5, o9, o13};
  float* cur = a;
  float* tmp = b;
  float* dst = c;
  for (int pass = 0; pass < 3; pass++) {
    for (int i = threadIdx.x; i < HW * SP_CC; i += blockDim.x) {
      const int ch = i % SP_CC, pix = i / SP_CC;
      const int h = pix / W, w = pix - h * W;
      float m = -INFINITY;
#pragma unroll
      for (int d = -2; d <= 2; d++) {
        const int ww = w + d;
        if (ww >= 0 && ww < W) m = fmaxf(m, cur[(h * W + ww) * SP_CC + ch]);
      }
      tmp[i] = m;
    }
    __syncthreads();
    T* o = reinterpret_cast<T*>(outs[pass].base);
    for (int i = threadIdx.x; i < HW * SP_CC; i += blockDim.x) {
      const int ch = i % SP_CC, pix = i / SP_CC;
      const int h = pix / W, w = pix - h * W;
      float m = -INFINITY;
#pragma unroll
      for (int d = -2; d <= 2; d++) {
        const int hh = h + d;
        if (hh >= 0 && hh < H) m = fmaxf(m, tmp[(hh * W + w) * SP_CC + ch]);
      }
      dst[i] = m;
      if (ch < cc)
        o[((size_t)n * HW + pix) * outs[pass].pitch + outs[pass].coff + c0 + ch] = from_f<T>(m);
    }
    __syncthreads();
    float* t = cur; cur = dst; dst = t;  // next pass pools the freshly pooled map
  }
}

// fp16 fast path: one CTA per (image, 8-channel chunk); a thread owns whole pixels as one 16-byte vector
// (4 x half2), separable 5x5 max = row pass + column pass through two smem planes, three cascaded pools.
__device__ __forceinline__ int4 hmax8(const int4& x, const int4& y) {
  int4 r;
  const __half2* a = reinterpret_cast<const __half2*>(&x);
  const __half2* b = reinterpret_cast<const __half2*>(&y);
  __half2* o = reinterpret_cast<__half2*>(&r);
#pragma unroll
  for (int j = 0; j < 4; j++) o[j] = __hmax2(a[j], b[j]);
  return r;
}

__global__ void __launch_bounds__(512) sppf_pool_h8_kernel(View in, View o5, View o9, View o13) {
  extern __shared__ __align__(16) int4 sp8[];
  const int H = in.H, W = in.W, HW = H * W;
  int4* cur = sp8;
  int4* tmp = sp8 + HW;
  const int n = blockIdx.y, c0 = blockIdx.x * 8;
  pdl_trigger();
  pdl_wait();
  const __half* src = reinterpret_cast<const __half*>(in.base) + (size_t)n * HW * in.pitch + in.coff + c0;
  for (int p = threadIdx.x; p < HW; p += blockDim.x) cur[p] = *reinterpret_cast<const int4*>(src + (size_t)p * in.pitch);
  __syncthreads();
#pragma unroll
  for (int pass = 0; pass < 3; pass++) {
    const View& ov = pass == 0 ? o5 : (pass == 1 ? o9 : o13);
    for (int p = threadIdx.x; p < HW; p += blockDim.x) {
      const int h = p / W, w = p - h * W;
      int4 m = cur[p];
#pragma unroll
      for (int d = -2; d <= 2; d++)
        if (d != 0 && w + d >= 0 && w + d < W) m = hmax8(m, cur[p + d]);
      tmp[p] = m;
    }
    __syncthreads();
    __half* dst = reinterpret_cast<__half*>(ov.base) + (size_t)n * HW * ov.pitch + ov.coff + c0;
    for (int p = threadIdx.x; p < HW; p += blockDim.x) {
      const int h = p / W;
      int4 m = tmp[p];
#pragma unroll
      for (int d = -2; d <= 2; d++)
        if (d != 0 && h + d >= 0 && h + d < H) m = hmax8(m, tmp[p + d * W]);
      cur[p] = m;  // safe: the column pass reads tmp only
      *reinterpret_cast<int4*>(dst + (size_t)p * ov.pitch) = m;
    }
    __syncthreads();
  }
}

template <typename T>
int launch_sppf_pool(const View& in, const View& o5, const View& o9, const View& o13, int B,
                     cudaStream_t s) {
  if (sizeof(T) == 2 && in.C % 8 == 0 && in.coff % 8 == 0 && in.pitch % 8 == 0 && o5.coff % 8 == 0 && o5.pitch % 8 == 0 &&
      o9.coff % 8 == 0 && o13.coff % 8 == 0 && (size_t)2 * in.H * in.W * 16 <= 48 * 1024) {
    const int HW = in.H * in.W;
    const int threads = std::min(512, (HW + 31) / 32 * 32);
    YB_CUDA_CHECK(launch_pdl(sppf_pool_h8_kernel, dim3(in.C / 8, B), dim3(threads), (size_t)2 * HW * 16, s, in, o5, o9, o13));
    return 0;
  }
  const size_t smem = (size_t)3 * in.H * in.W * SP_CC * sizeof(float);
  if (smem > 200 * 1024) {
    set_error("sppf_pool: feature map too large for the shared-memory kernel");
    return YB_ERR_SHAPE;
  }
  YB_CUDA_CHECK(smem_limit((const void*)sppf_pool_kernel<T>, smem, false));
  dim3 grid((in.C + SP_CC - 1) / SP_CC, B);
  sppf_pool_kernel<T><<<grid, 256, smem, s>>>(in, o5, o9, o13);
  YB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
template int launch_sppf_pool<float>(const View&, const View&, const View&, const View&, int, cudaStream_t);
template int launch_sppf_pool<__half>(const View&, const View&, const View&, const View&, int, cudaStream_t);

// ------------------------------------------------------------------------------------------
// nn.Upsample(scale 2, nearest) written straight into a concat slice (Yolo.cs:70,74).
// ------------------------------------------------------------------------------------------
template <typename T, typename V>
__global__ void upsample2x_kernel(View in, View out, size_t total, int vec) {
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cv = in.C / vec;
  const int c = (idx % cv) * vec;
  size_t pix = idx / cv;
  const int w = pix % out.W;
  const int h = (pix / out.W) % out.H;
  const int n = pix / ((size_t)out.W * out.H);
  const T* src = reinterpret_cast<const T*>(in.base) +
                 ((size_t)(n * in.H + (h >> 1)) * in.W + (w >> 1)) * in.pitch + in.coff + c;
  T* dst = reinterpret_cast<T*>(out.base) + pix * out.pitch + out.coff + c;
  *reinterpret_cast<V*>(dst) = *reinterpret_cast<const V*>(src);
}

// Row-structured version for 16-byte vectors: one block per input row, every vector is read once and stored to its
// 2 x 2 output pixels; 32-bit index math only (the per-element kernel above spends its time in 64-bit divisions:
// 2.5 TB/s on the 40x40 -> 80x80 layer of v8n, this one is bandwidth-bound).
__global__ void __launch_bounds__(256) upsample2x_rows_kernel(const int4* __restrict__ in, int4* __restrict__ out, int Hin, int Win,
                                                              int cv, int in_pitch_v, int out_pitch_v) {
  const int row = blockIdx.x;  // n * Hin + h
  const int n = row / Hin, h = row - n * Hin;
  const int4* src = in + (size_t)row * Win * in_pitch_v;
  int4* dst0 = out + ((size_t)(n * 2 * Hin + 2 * h) * 2 * Win) * out_pitch_v;
  int4* dst1 = dst0 + (size_t)2 * Win * out_pitch_v;
  for (int i = threadIdx.x; i < Win * cv; i += blockDim.x) {
    const int w = i / cv, c = i - w * cv;
    const int4 v = __ldg(src + w * in_pitch_v + c);
    const int o = 2 * w * out_pitch_v + c;
    dst0[o] = v;
    dst0[o + out_pitch_v] = v;
    dst1[o] = v;
    dst1[o + out_pitch_v] = v;
  }
}

template <typename T>
int launch_upsample2x(const View& in, const View& out, int B, cudaStream_t s) {
  // widest vector such that every slice start stays aligned
  int vec = 16 / (int)sizeof(T);
  while (vec > 1 && (in.C % vec || in.coff % vec || in.pitch % vec || out.coff % vec || out.pitch % vec)) vec >>= 1;
  if (vec * (int)sizeof(T) == 16) {
    const int4* src = reinterpret_cast<const int4*>(reinterpret_cast<const T*>(in.base) + in.coff);
    int4* dst = reinterpret_cast<int4*>(reinterpret_cast<T*>(out.base) + out.coff);
    upsample2x_rows_kernel<<<B * in.H, 256, 0, s>>>(src, dst, in.H, in.W, in.C / vec, in.pitch / vec, out.pitch / vec);
    YB_CUDA_CHECK(cudaGetLastError());
    return 0;
  }
  const size_t total = (size_t)B * out.H * out.W * (in.C / vec);
  const unsigned blocks = (unsigned)((total + 255) / 256);
  const int bytes = vec * (int)sizeof(T);
  if (bytes == 8) upsample2x_kernel<T, int2><<<blocks, 256, 0, s>>>(in, out, total, vec);
  else if (bytes == 4) upsample2x_kernel<T, int><<<blocks, 256, 0, s>>>(in, out, total, vec);
  else upsample2x_kernel<T, T><<<blocks, 256, 0, s>>>(in, out, total, vec);
  YB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
template int launch_upsample2x<float>(const View&, const View&, int, cudaStream_t);
template int launch_upsample2x<__half>(const View&, const View&, int, cudaStream_t);

// ------------------------------------------------------------------------------------------
// Network input (B,3,H,W) NCHW u8|f16|f32 -> NHWC T.  u8 is divided by 255 in fp32 exactly as
// Detector.cs:41 does (`pad(...) / 255.0f`).
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float load_input(const void* in, int dtype, size_t i) {
  if (dtype == YB_U8) return __fdiv_rn((float)reinterpret_cast<const uint8_t*>(in)[i], 255.0f);
  if (dtype == YB_F16) return __half2float(reinterpret_cast<const __half*>(in)[i]);
  return reinterpret_cast<const float*>(in)[i];
}

template <typename T>
__global__ void input_to_nhwc_kernel(const void* in, int dtype, View out, size_t npix_total, int src_H, int src_W) {
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= npix_total) return;
  const size_t HW = (size_t)out.H * out.W, sHW = (size_t)src_H * src_W;
  const size_t n = idx / HW, pix = idx - n * HW;
  const int y = (int)(pix / out.W), x = (int)(pix - (size_t)y * out.W);
  T* dst = reinterpret_cast<T*>(out.base) + idx * out.pitch + out.coff;
  // right / bottom padding with 114 before the /255 (Detector.cs:35-41): pad(x, 114) / 255
  const bool inside = y < src_H && x < src_W;
#pragma unroll
  for (int c = 0; c < 3; c++)
    dst[c] = from_f<T>(inside ? load_input(in, dtype, (n * 3 + c) * sHW + (size_t)y * src_W + x) : __fdiv_rn(114.0f, 255.0f));
}

template <typename T>
int launch_input_to_nhwc(const void* in, int in_dtype, const View& out, int B, cudaStream_t s, int src_H, int src_W) {
  const size_t total = (size_t)B * out.H * out.W;
  if (src_H <= 0) src_H = out.H;
  if (src_W <= 0) src_W = out.W;
  input_to_nhwc_kernel<T><<<(unsigned)((total + 255) / 256), 256, 0, s>>>(in, in_dtype, out, total, src_H, src_W);
  YB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
template int launch_input_to_nhwc<float>(const void*, int, const View&, int, cudaStream_t, int, int);
template int launch_input_to_nhwc<__half>(const void*, int, const View&, int, cudaStream_t, int, int);

template <typename T>
__global__ void view_to_nchw_kernel(View in, float* out, size_t total) {
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const size_t HW = (size_t)in.H * in.W;
  const size_t pix = idx % HW;
  const int c = (idx / HW) % in.C;
  const size_t n = idx / (HW * in.C);
  out[idx] = to_f<T>(reinterpret_cast<const T*>(in.base)[(n * HW + pix) * in.pitch + in.coff + c]);
}

template <typename T>
int launch_view_to_nchw_f32(const View& in, float* out, int B, cudaStream_t s) {
  const size_t total = (size_t)B * in.C * in.H * in.W;
  view_to_nchw_kernel<T><<<(unsigned)((total + 255) / 256), 256, 0, s>>>(in, out, total);
  YB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
template int launch_view_to_nchw_f32<float>(const View&, float*, int, cudaStream_t);
template int launch_view_to_nchw_f32<__half>(const View&, float*, int, cudaStream_t);

// ------------------------------------------------------------------------------------------
// Head decode for one pyramid level.  One thread per (image, anchor):
//   DFL   (Block.cs:44): softmax over the 16 bins of each side, expectation with weights 0..15
//   boxes (Tal.cs:338-356, Head.cs:221): anchor = (x+0.5, y+0.5); x1y1 = a - lt; x2y2 = a + rb;
//         xywh = ((x1y1+x2y2)/2, x2y2-x1y1) * stride
//   cls   (Head.cs:207): sigmoid
// Output layout is the reference's (B, 4+nc[+nm], A): channel-major, anchors contiguous, so the
// per-channel stores of a warp are coalesced.
// ------------------------------------------------------------------------------------------
template <typename T>
__global__ void decode_level_kernel(View box, View cls, View coef, int has_coef, int B, int nc, int nm,
                                    int reg_max, float stride, int a0, int A, int Ctot, float* pred) {
  const int HW = box.H * box.W;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)B * HW) return;
  const int n = idx / HW, i = idx - (size_t)n * HW;
  const int y = i / box.W, x = i - y * box.W;
  const T* bp = reinterpret_cast<const T*>(box.base) + idx * box.pitch + box.coff;
  float* out = pred + (size_t)n * Ctot * A + a0 + i;
  float d[4];
  for (int sd = 0; sd < 4; sd++) {
    float mx = -INFINITY;
    for (int k = 0; k < reg_max; k++) mx = fmaxf(mx, to_f<T>(bp[sd * reg_max + k]));
    float sum = 0.f, ex = 0.f;
    for (int k = 0; k < reg_max; k++) {
      const float e = expf(to_f<T>(bp[sd * reg_max + k]) - mx);
      sum += e;
      ex = fmaf(e, (float)k, ex);
    }
    d[sd] = ex / sum;
  }
  const float ax = (float)x + 0.5f, ay = (float)y + 0.5f;
  const float x1 = ax - d[0], y1 = ay - d[1], x2 = ax + d[2], y2 = ay + d[3];
  out[0 * (size_t)A] = ((x1 + x2) / 2.0f) * stride;
  out[1 * (size_t)A] = ((y1 + y2) / 2.0f) * stride;
  out[2 * (size_t)A] = (x2 - x1) * stride;
  out[3 * (size_t)A] = (y2 - y1) * stride;
  const T* cp = reinterpret_cast<const T*>(cls.base) + idx * cls.pitch + cls.coff;
  for (int c = 0; c < nc; c++) out[(size_t)(4 + c) * A] = 1.0f / (1.0f + expf(-to_f<T>(cp[c])));
  if (has_coef) {
    const T* mp = reinterpret_cast<const T*>(coef.base) + idx * coef.pitch + coef.coff;
    for (int c = 0; c < nm; c++) out[(size_t)(4 + nc + c) * A] = to_f<T>(mp[c]);
  }
}

template <typename T>
int launch_decode_level(const View& box, const View& cls, const View* coef, int B, int nc, int nm,
                        int reg_max, float stride, int a0, int A, int Ctot, float* pred, cudaStream_t s) {
  const size_t total = (size_t)B * box.H * box.W;
  View cf = coef ? *coef : View();
  decode_level_kernel<T><<<(unsigned)((total + 127) / 128), 128, 0, s>>>(box, cls, cf, coef != nullptr, B, nc, nm,
                                                                        reg_max, stride, a0, A, Ctot, pred);
  YB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
template int launch_decode_level<float>(const View&, const View&, const View*, int, int, int, int, float, int, int, int, float*, cudaStream_t);
template int launch_decode_level<__half>(const View&, const View&, const View*, int, int, int, int, float, int, int, int, float*, cudaStream_t);

// proto (B,h,w,C) NHWC T -> (B,C,h,w) fp32 through a 32x33 shared tile (coalesced both ways)
template <typename T>
__global__ void proto_out_kernel(View in, float* out, int HW) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;  // 32 x 8
  const T* src = reinterpret_cast<const T*>(in.base);
  for (int r = ty; r < 32; r += 8) {
    const int pix = p0 + r, c = c0 + tx;
    tile[r][tx] = (pix < HW && c < in.C) ? to_f<T>(src[((size_t)n * HW + pix) * in.pitch + in.coff + c]) : 0.f;
  }
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {
    const int c = c0 + r, pix = p0 + tx;
    if (c < in.C && pix < HW) out[((size_t)n * in.C + c) * HW + pix] = tile[tx][r];
  }
}

template <typename T>
int launch_proto_out(const View& in, float* out, int B, cudaStream_t s) {
  const int HW = in.H * in.W;
  dim3 grid((HW + 31) / 32, (in.C + 31) / 32, B);
  proto_out_kernel<T><<<grid, dim3(32, 8), 0, s>>>(in, out, HW);
  YB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
template int launch_proto_out<float>(const View&, float*, int, cudaStream_t);
template int launch_proto_out<__half>(const View&, float*, int, cudaStream_t);

}  // namespace yb

namespace yb {

// ------------------------------------------------------------------------------------------
// ConvTranspose2d(c, c, 2, 2, 0) of Proto (Block.cs:69,82) = one 1x1 conv to 4*c channels
// (phase-major: oc = (i*2+j)*c + co) followed by this pixel shuffle:
//   out[n, 2h+i, 2w+j, co] = in[n, h, w, (i*2+j)*c + co]
// ------------------------------------------------------------------------------------------
template <typename T, typename V>
__global__ void pixel_shuffle2_kernel(View in, View out, size_t total, int vec) {
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cv = out.C / vec;
  const int c = (idx % cv) * vec;
  size_t pix = idx / cv;
  const int w = pix % out.W;
  const int h = (pix / out.W) % out.H;
  const int n = pix / ((size_t)out.W * out.H);
  const int ph = ((h & 1) * 2 + (w & 1)) * out.C;
  const T* src = reinterpret_cast<const T*>(in.base) +
                 ((size_t)(n * in.H + (h >> 1)) * in.W + (w >> 1)) * in.pitch + in.coff + ph + c;
  T* dst = reinterpret_cast<T*>(out.base) + pix * out.pitch + out.coff + c;
  *reinterpret_cast<V*>(dst) = *reinterpret_cast<const V*>(src);
}

template <typename T>
int launch_pixel_shuffle2(const View& in, const View& out, int B, cudaStream_t s) {
  int vec = 16 / (int)sizeof(T);
  while (vec > 1 && (out.C % vec || in.coff % vec || in.pitch % vec || out.coff % vec || out.pitch % vec)) vec >>= 1;
  const size_t total = (size_t)B * out.H * out.W * (out.C / vec);
  const unsigned blocks = (unsigned)((total + 255) / 256);
  const int bytes = vec * (int)sizeof(T);
  if (bytes == 16) pixel_shuffle2_kernel<T, int4><<<blocks, 256, 0, s>>>(in, out, total, vec);
  else if (bytes == 8) pixel_shuffle2_kernel<T, int2><<<blocks, 256, 0, s>>>(in, out, total, vec);
  else if (bytes == 4) pixel_shuffle2_kernel<T, int><<<blocks, 256, 0, s>>>(in, out, total, vec);
  else pixel_shuffle2_kernel<T, T><<<blocks, 256, 0, s>>>(in, out, total, vec);
  YB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
template int launch_pixel_shuffle2<float>(const View&, const View&, int, cudaStream_t);
template int launch_pixel_shuffle2<__half>(const View&, const View&, int, cudaStream_t);

}  // namespace yb
