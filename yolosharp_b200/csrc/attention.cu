// C2PSA attention core (Block.cs:752-809), forward and backward, for the inference engine and the training step:
//   attn = softmax_j(q_i . k_j * scale);  out_i = sum_j attn_ij v_j
// Each pass has one general kernel and one register-blocked kernel for kd = 32, hd = 64 (every YOLOv11 size:
// num_heads = c / 64, key_dim = 32; N = 400 tokens at 640 x 640).  The forward pair is shared by the engine (T = float /
// __half, q | k | v interleaved per head in the qkv conv output) and the training step (fp32, separate q, k, v); AttnIO
// describes where token t of head h of image b lives.  The backward (training only, fp32) recomputes the forward for its
// row statistics.  Everything is deterministic: per-row reductions in a fixed order, no floating-point atomics.
#include <cmath>

#include "common.cuh"

namespace yb {

struct AttnIO {
  const void *q, *k, *v;             // element type T
  long long in_tok, in_img;          // element strides between tokens / images of q and k
  long long v_tok, v_img;            // the same for v
  long long q_head, k_head, v_head;  // element offset of head h: h * q_head etc.
  void* out;                         // type T; token t of head h at out + b * out_img + t * out_tok + h * hd
  long long out_tok, out_img;
  void* vout;                        // optional dense copy of v (same addressing as out), type T
  float *row_max, *row_sum;          // optional (B, nh, N) fp32 softmax statistics for the backward pass
};

// ------------------------------------------------------------------------------------------
// General forward: one warp per query row, K and V streamed through shared memory in blocks of 32 keys.
// ------------------------------------------------------------------------------------------
constexpr int AG_WARPS = 8;
template <typename T>
__global__ void __launch_bounds__(256) attention_kernel(AttnIO io, int N, int nh, int kd, int hd, float scale) {
  extern __shared__ float at_smem[];  // per warp: scores[N]; shared: K block [32][kd+1], V block [32][hd]
  const int b = blockIdx.z, head = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nwarps = blockDim.x >> 5;
  const T* qb = reinterpret_cast<const T*>(io.q) + (size_t)b * io.in_img + (size_t)head * io.q_head;
  const T* kb = reinterpret_cast<const T*>(io.k) + (size_t)b * io.in_img + (size_t)head * io.k_head;
  const T* vb = reinterpret_cast<const T*>(io.v) + (size_t)b * io.v_img + (size_t)head * io.v_head;
  float* sc = at_smem + (size_t)warp * N;
  float* kblk = at_smem + (size_t)nwarps * N;
  float* vblk = kblk + 32 * (kd + 1);
  const int i = blockIdx.x * nwarps + warp;  // query row of this warp
  const bool active = i < N;
  // q_i in registers (kd <= 64: up to 2 per lane)
  float q0 = 0.f, q1 = 0.f;
  if (active) {
    if (lane < kd) q0 = to_f<T>(qb[(size_t)i * io.in_tok + lane]);
    if (lane + 32 < kd) q1 = to_f<T>(qb[(size_t)i * io.in_tok + lane + 32]);
  }
  // pass 1: scores
  for (int j0 = 0; j0 < N; j0 += 32) {
    __syncthreads();
    for (int t = threadIdx.x; t < 32 * kd; t += blockDim.x) {
      const int jj = t / kd, d = t - jj * kd;
      kblk[jj * (kd + 1) + d] = (j0 + jj < N) ? to_f<T>(kb[(size_t)(j0 + jj) * io.in_tok + d]) : 0.f;
    }
    __syncthreads();
    if (active) {
      // lane = key j0+lane: dot(q_i, k_j) with q broadcast by shuffles
      float acc = 0.f;
      for (int d = 0; d < kd; d++) {
        const float qd = __shfl_sync(0xffffffffu, d < 32 ? q0 : q1, d & 31);
        acc = fmaf(qd, kblk[lane * (kd + 1) + d], acc);
      }
      if (j0 + lane < N) sc[j0 + lane] = acc * scale;
    }
  }
  __syncwarp();
  float mx = -INFINITY;
  if (active)
    for (int j = lane; j < N; j += 32) mx = fmaxf(mx, sc[j]);
  for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
  if (active)
    for (int j = lane; j < N; j += 32) {
      const float e = expf(sc[j] - mx);
      sc[j] = e;
      sum += e;
    }
  for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float inv = 1.0f / sum;
  __syncwarp();
  // pass 2: out_i[d] = sum_j p_j v_j[d]; lane owns d = lane, lane+32, ...
  float o0 = 0.f, o1 = 0.f, o2 = 0.f, o3 = 0.f;
  for (int j0 = 0; j0 < N; j0 += 32) {
    __syncthreads();
    for (int t = threadIdx.x; t < 32 * hd; t += blockDim.x) {
      const int jj = t / hd, d = t - jj * hd;
      vblk[jj * hd + d] = (j0 + jj < N) ? to_f<T>(vb[(size_t)(j0 + jj) * io.v_tok + d]) : 0.f;
    }
    __syncthreads();
    if (active) {
      const int jn = min(32, N - j0);
      for (int jj = 0; jj < jn; jj++) {
        const float pj = sc[j0 + jj];
        if (lane < hd) o0 = fmaf(pj, vblk[jj * hd + lane], o0);
        if (lane + 32 < hd) o1 = fmaf(pj, vblk[jj * hd + lane + 32], o1);
        if (lane + 64 < hd) o2 = fmaf(pj, vblk[jj * hd + lane + 64], o2);
        if (lane + 96 < hd) o3 = fmaf(pj, vblk[jj * hd + lane + 96], o3);
      }
    }
  }
  if (!active) return;
  const size_t orow = (size_t)b * io.out_img + (size_t)i * io.out_tok + (size_t)head * hd;
  T* op = reinterpret_cast<T*>(io.out) + orow;
  T* vp = io.vout ? reinterpret_cast<T*>(io.vout) + orow : nullptr;
  const T* vsrc = vb + (size_t)i * io.v_tok;
  const float ov[4] = {o0, o1, o2, o3};
#pragma unroll
  for (int r = 0; r < 4; r++) {
    const int d = lane + 32 * r;
    if (d < hd) {
      op[d] = from_f<T>(ov[r] * inv);
      if (vp) vp[d] = vsrc[d];
    }
  }
  if (lane == 0 && io.row_max) {
    io.row_max[((size_t)b * nh + head) * N + i] = mx;
    io.row_sum[((size_t)b * nh + head) * N + i] = sum;
  }
}

// ------------------------------------------------------------------------------------------
// Register-blocked forward for kd = 32, hd = 64, used when a head's K and V fit in shared memory (N <= 424 tokens:
// every 640 x 640 model).  The general kernel above re-streams K and V through shared memory for every 8 query rows
// (6 400 CTAs x 77 KB and 100 block-wide barriers each for YOLOv11s at batch 32).  Scalar shared-memory reads would
// make a tiled version shared-memory bound (three LDS per two FMAs).  This one is register-blocked:
//   * a CTA (16 warps) owns 32 query rows of one (head, image); K (row stride 36 floats) and V (stride 64) stay resident as fp32
//   * scores: a warp owns 2 query rows, held in 64 registers; a lane owns one key per block of 32 and reads its K row
//     with 8 conflict-free LDS.128 -> 64 FMAs per 8 loads
//   * P.V: a lane owns channels 2*lane, 2*lane+1 for both rows; per 4 keys: 4 LDS.64 of V + 2 broadcast LDS.128 of P
//     for 16 FMAs
// Per-output summation order is sequential over d, then over j.
// ------------------------------------------------------------------------------------------
constexpr int ATI_T = 32, ATI_KD = 32, ATI_HD = 64, ATI_LDK = 36, ATI_THREADS = 512;  // 16 warps x 2 query rows
__device__ __forceinline__ float4 lds4(const float* p) { return *reinterpret_cast<const float4*>(p); }
// four consecutive elements (16 / 8 bytes, aligned) as fp32: one vector load instead of four scalar ones - the scalar
// fill of K and V made every warp instruction touch 16 sectors for 128 useful bytes and cost 2/3 of the kernel
template <typename T> __device__ __forceinline__ float4 ld4(const T* p);
template <> __device__ __forceinline__ float4 ld4<float>(const float* p) { return *reinterpret_cast<const float4*>(p); }
template <> __device__ __forceinline__ float4 ld4<__half>(const __half* p) {
  const uint2 u = *reinterpret_cast<const uint2*>(p);
  const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
  return make_float4(a.x, a.y, b.x, b.y);
}
template <typename T> __device__ __forceinline__ void cp4(T* dst, const T* src);
template <> __device__ __forceinline__ void cp4<float>(float* dst, const float* src) { *reinterpret_cast<float4*>(dst) = *reinterpret_cast<const float4*>(src); }
template <> __device__ __forceinline__ void cp4<__half>(__half* dst, const __half* src) { *reinterpret_cast<uint2*>(dst) = *reinterpret_cast<const uint2*>(src); }

template <typename T>
__global__ void __launch_bounds__(ATI_THREADS, 1) attention_tiled_32x64_kernel(AttnIO io, int N, int nh, float scale) {
  extern __shared__ __align__(16) float at_smem[];
  const int NK = (N + 31) & ~31, NP = (N + 3) & ~3;
  float* Ks = at_smem;                          // [NK][36], rows >= N zero
  float* Vs = Ks + (size_t)NK * ATI_LDK;        // [NP][64], rows >= N zero
  float* Qs = Vs + (size_t)NP * ATI_HD;         // [16][32]
  float* Ps = Qs + ATI_T * ATI_KD;              // [16][NP]
  const int i0 = blockIdx.x * ATI_T, head = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const T* qb = reinterpret_cast<const T*>(io.q) + (size_t)b * io.in_img + (size_t)head * io.q_head;
  const T* kb = reinterpret_cast<const T*>(io.k) + (size_t)b * io.in_img + (size_t)head * io.k_head;
  const T* vb = reinterpret_cast<const T*>(io.v) + (size_t)b * io.v_img + (size_t)head * io.v_head;
  T* vo = reinterpret_cast<T*>(io.vout);
  // fill: 4 channels per thread and step, 8 independent vector loads in flight per thread (with one CTA of 8 warps per
  // SM a load-convert-store loop exposes the full L2 latency on every iteration: 38 iterations x ~700 cycles was 2/3 of
  // the kernel)
  constexpr int U = 8;
  for (int t0 = threadIdx.x; t0 < NK * (ATI_KD / 4); t0 += ATI_THREADS * U) {
    float4 f[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const int t = t0 + u * ATI_THREADS, j = t >> 3, d = (t & 7) * 4;
      f[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (t < NK * (ATI_KD / 4) && j < N) f[u] = ld4<T>(kb + (size_t)j * io.in_tok + d);
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      const int t = t0 + u * ATI_THREADS, j = t >> 3, d = (t & 7) * 4;
      if (t < NK * (ATI_KD / 4)) *reinterpret_cast<float4*>(Ks + (size_t)j * ATI_LDK + d) = f[u];
    }
  }
  for (int t0 = threadIdx.x; t0 < NP * (ATI_HD / 4); t0 += ATI_THREADS * U) {
    float4 f[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const int t = t0 + u * ATI_THREADS, j = t >> 4, d = (t & 15) * 4;
      f[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (t < NP * (ATI_HD / 4) && j < N) {
        f[u] = ld4<T>(vb + (size_t)j * io.v_tok + d);
      }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      const int t = t0 + u * ATI_THREADS, j = t >> 4, d = (t & 15) * 4;
      if (t < NP * (ATI_HD / 4)) *reinterpret_cast<float4*>(Vs + (size_t)j * ATI_HD + d) = f[u];
    }
  }
  // the dense copy of v that the positional-encoding conv reads: this CTA's 32 rows, one vector per thread.  (Inside the
  // fill loop above these stores would sit between the batched loads and each wait for its own load.)
  if (vo) {
    const int r = threadIdx.x >> 4, d = (threadIdx.x & 15) * 4, j = i0 + r;
    if (j < N) cp4<T>(vo + (size_t)b * io.out_img + (size_t)j * io.out_tok + head * ATI_HD + d, vb + (size_t)j * io.v_tok + d);
  }
  for (int t = threadIdx.x; t < ATI_T * ATI_KD; t += ATI_THREADS) {
    const int r = t >> 5, d = t & 31;
    Qs[t] = (i0 + r < N) ? to_f<T>(qb[(size_t)(i0 + r) * io.in_tok + d]) : 0.f;
  }
  __syncthreads();
  const int r0 = warp * 2, r1 = r0 + 1;
  float* p0 = Ps + (size_t)r0 * NP;
  float* p1 = Ps + (size_t)r1 * NP;
  float q0[ATI_KD], q1[ATI_KD];
#pragma unroll
  for (int d = 0; d < ATI_KD; d += 4) {
    const float4 a = lds4(Qs + r0 * ATI_KD + d), c = lds4(Qs + r1 * ATI_KD + d);
    q0[d] = a.x; q0[d + 1] = a.y; q0[d + 2] = a.z; q0[d + 3] = a.w;
    q1[d] = c.x; q1[d + 1] = c.y; q1[d + 2] = c.z; q1[d + 3] = c.w;
  }
  float m0 = -INFINITY, m1 = -INFINITY;
  for (int j = lane; j < NK; j += 32) {
    const float* kr = Ks + (size_t)j * ATI_LDK;
    float s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int d = 0; d < ATI_KD; d += 4) {
      const float4 kv = lds4(kr + d);
      s0 = fmaf(q0[d], kv.x, s0); s1 = fmaf(q1[d], kv.x, s1);
      s0 = fmaf(q0[d + 1], kv.y, s0); s1 = fmaf(q1[d + 1], kv.y, s1);
      s0 = fmaf(q0[d + 2], kv.z, s0); s1 = fmaf(q1[d + 2], kv.z, s1);
      s0 = fmaf(q0[d + 3], kv.w, s0); s1 = fmaf(q1[d + 3], kv.w, s1);
    }
    if (j < N) {
      s0 *= scale; s1 *= scale;
      p0[j] = s0; p1[j] = s1;
      m0 = fmaxf(m0, s0); m1 = fmaxf(m1, s1);
    } else if (j < NP) {
      p0[j] = -INFINITY; p1[j] = -INFINITY;  // exp -> 0: padded keys contribute nothing
    }
  }
  for (int o = 16; o; o >>= 1) { m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, o)); m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, o)); }
  float l0 = 0.f, l1 = 0.f;
  for (int j = lane; j < NP; j += 32) {
    const float e0 = expf(p0[j] - m0), e1 = expf(p1[j] - m1);
    p0[j] = e0; p1[j] = e1;
    l0 += e0; l1 += e1;
  }
  for (int o = 16; o; o >>= 1) { l0 += __shfl_xor_sync(0xffffffffu, l0, o); l1 += __shfl_xor_sync(0xffffffffu, l1, o); }
  __syncwarp();
  float a00 = 0.f, a01 = 0.f, a10 = 0.f, a11 = 0.f;
  const float* vcol = Vs + 2 * lane;
  for (int j = 0; j < NP; j += 4) {
    const float4 pa = lds4(p0 + j), pb = lds4(p1 + j);
    const float2 v0 = *reinterpret_cast<const float2*>(vcol + (size_t)j * ATI_HD);
    const float2 v1 = *reinterpret_cast<const float2*>(vcol + (size_t)(j + 1) * ATI_HD);
    const float2 v2 = *reinterpret_cast<const float2*>(vcol + (size_t)(j + 2) * ATI_HD);
    const float2 v3 = *reinterpret_cast<const float2*>(vcol + (size_t)(j + 3) * ATI_HD);
    a00 = fmaf(pa.x, v0.x, a00); a01 = fmaf(pa.x, v0.y, a01); a10 = fmaf(pb.x, v0.x, a10); a11 = fmaf(pb.x, v0.y, a11);
    a00 = fmaf(pa.y, v1.x, a00); a01 = fmaf(pa.y, v1.y, a01); a10 = fmaf(pb.y, v1.x, a10); a11 = fmaf(pb.y, v1.y, a11);
    a00 = fmaf(pa.z, v2.x, a00); a01 = fmaf(pa.z, v2.y, a01); a10 = fmaf(pb.z, v2.x, a10); a11 = fmaf(pb.z, v2.y, a11);
    a00 = fmaf(pa.w, v3.x, a00); a01 = fmaf(pa.w, v3.y, a01); a10 = fmaf(pb.w, v3.x, a10); a11 = fmaf(pb.w, v3.y, a11);
  }
  const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
  T* ob = reinterpret_cast<T*>(io.out) + (size_t)b * io.out_img + head * ATI_HD + 2 * lane;
  if (i0 + r0 < N) { T* o = ob + (size_t)(i0 + r0) * io.out_tok; o[0] = from_f<T>(a00 * inv0); o[1] = from_f<T>(a01 * inv0); }
  if (i0 + r1 < N) { T* o = ob + (size_t)(i0 + r1) * io.out_tok; o[0] = from_f<T>(a10 * inv1); o[1] = from_f<T>(a11 * inv1); }
  if (lane == 0 && io.row_max) {
    if (i0 + r0 < N) { io.row_max[((size_t)b * nh + head) * N + i0 + r0] = m0; io.row_sum[((size_t)b * nh + head) * N + i0 + r0] = l0; }
    if (i0 + r1 < N) { io.row_max[((size_t)b * nh + head) * N + i0 + r1] = m1; io.row_sum[((size_t)b * nh + head) * N + i0 + r1] = l1; }
  }
}

// ------------------------------------------------------------------------------------------
// Forward launch: the one rule the engine and the training step share.
// ------------------------------------------------------------------------------------------
// The limits every attention call is held to are those of the general kernel (the register-blocked one takes a subset
// of its shapes): key_dim <= 64 (q_i sits in two registers per lane), head_dim <= 128 (four accumulators per lane) and
// 8 N + 32 (key_dim + 1) + 32 head_dim floats of shared memory <= 200 KiB, i.e. N <= 6 012 tokens at key_dim 32,
// head_dim 64.  The backward recomputes the forward, and its kernels need less shared memory, so the same limits hold.
constexpr size_t AG_SMEM_MAX = 200 * 1024;
static size_t ag_smem_bytes(int N, int kd, int hd) { return ((size_t)AG_WARPS * N + 32 * (kd + 1) + 32 * (size_t)hd) * sizeof(float); }
static int attention_check(int B, int N, int nh, int kd, int hd) {
  if (B <= 0 || N <= 0 || nh <= 0 || kd <= 0 || hd <= 0) { set_error("attention: bad shape"); return YB_ERR_SHAPE; }
  if (kd > 64 || hd > 128) {
    set_error("attention: key_dim <= 64 and head_dim <= 128 supported, got " + std::to_string(kd) + " / " + std::to_string(hd));
    return YB_ERR_SHAPE;
  }
  if (ag_smem_bytes(N, kd, hd) > AG_SMEM_MAX) {
    const size_t max_n = (AG_SMEM_MAX / sizeof(float) - 32 * (kd + 1) - 32 * (size_t)hd) / AG_WARPS;
    set_error("attention: " + std::to_string(N) + " tokens exceed the shared-memory limit of " + std::to_string(max_n) +
              " at key_dim " + std::to_string(kd) + ", head_dim " + std::to_string(hd));
    return YB_ERR_SHAPE;
  }
  return 0;
}

static size_t ati_smem_bytes(int N) {
  const size_t NK = (N + 31) & ~31, NP = (N + 3) & ~3;
  return (NK * ATI_LDK + NP * ATI_HD + (size_t)ATI_T * ATI_KD + (size_t)ATI_T * NP) * sizeof(float);
}
// the register-blocked kernel reads k and v rows and writes the v copy as 4-element vectors
template <typename T>
static bool ati_vec4_ok(const AttnIO& io) {
  const uintptr_t p = (uintptr_t)io.k | (uintptr_t)io.v | (uintptr_t)io.out | (uintptr_t)io.vout;
  const long long st = io.in_tok | io.in_img | io.v_tok | io.v_img | io.k_head | io.v_head | io.out_tok | io.out_img;
  return p % (4 * sizeof(T)) == 0 && st % 4 == 0;
}

template <typename T>
static int attention_launch(const AttnIO& io, int B, int N, int nh, int kd, int hd, float scale, cudaStream_t s) {
  if (int rc = attention_check(B, N, nh, kd, hd)) return rc;
  if (kd == ATI_KD && hd == ATI_HD && ati_smem_bytes(N) <= 227 * 1024 && ati_vec4_ok<T>(io)) {
    YB_CUDA_CHECK(smem_limit((const void*)attention_tiled_32x64_kernel<T>, ati_smem_bytes(N), false));
    attention_tiled_32x64_kernel<T><<<dim3((N + ATI_T - 1) / ATI_T, nh, B), ATI_THREADS, ati_smem_bytes(N), s>>>(io, N, nh, scale);
  } else {
    YB_CUDA_CHECK(smem_limit((const void*)attention_kernel<T>, ag_smem_bytes(N, kd, hd), false));
    attention_kernel<T><<<dim3((N + AG_WARPS - 1) / AG_WARPS, nh, B), AG_WARPS * 32, ag_smem_bytes(N, kd, hd), s>>>(io, N, nh, kd, hd, scale);
  }
  YB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// engine: qkv is the NHWC output of the qkv conv, token t = pixel, channel = head*(2kd+hd) + [q | k | v].  Writes out
// (B,N,C) with channel head*hd + d, and the dense copy of v the positional-encoding depthwise conv needs
// (`pe(v.reshape(B,C,H,W))`).
template <typename T>
int launch_attention(const View& qkv, const View& out, const View& vout, int B, int nh, int kd, int hd, float scale,
                     cudaStream_t s) {
  if (vout.pitch != out.pitch) { set_error("attention: out and v copy must share their pitch"); return YB_ERR_SHAPE; }
  const int N = qkv.H * qkv.W;
  const T* base = reinterpret_cast<const T*>(qkv.base) + qkv.coff;
  AttnIO io;
  io.q = base; io.k = base + kd; io.v = base + 2 * kd;
  io.in_tok = io.v_tok = qkv.pitch; io.in_img = io.v_img = (long long)N * qkv.pitch;
  io.q_head = io.k_head = io.v_head = 2 * kd + hd;
  io.out = reinterpret_cast<T*>(out.base) + out.coff; io.out_tok = out.pitch; io.out_img = (long long)N * out.pitch;
  io.vout = reinterpret_cast<T*>(vout.base) + vout.coff;
  io.row_max = io.row_sum = nullptr;
  return attention_launch<T>(io, B, N, nh, kd, hd, scale, s);
}
template int launch_attention<float>(const View&, const View&, const View&, int, int, int, int, float, cudaStream_t);
template int launch_attention<__half>(const View&, const View&, const View&, int, int, int, int, float, cudaStream_t);

// training: q, k: (B, N, nh, kd); v, out: (B, N, nh, hd)
int attention_forward_f32(const float* q, const float* k, const float* v, int B, int N, int nh, int kd, int hd, float scale,
                          float* out, float* row_max, float* row_sum, cudaStream_t s) {
  AttnIO io;
  io.q = q; io.k = k; io.v = v;
  io.in_tok = (long long)nh * kd; io.in_img = (long long)N * nh * kd;
  io.v_tok = (long long)nh * hd; io.v_img = (long long)N * nh * hd;
  io.q_head = io.k_head = kd; io.v_head = hd;
  io.out = out; io.out_tok = (long long)nh * hd; io.out_img = (long long)N * nh * hd;
  io.vout = nullptr; io.row_max = row_max; io.row_sum = row_sum;
  return attention_launch<float>(io, B, N, nh, kd, hd, scale, s);
}

// ---------------------------------------------------------------------------------------------------------------
// General backward, one CTA per row: q, k, dq, dk (B, N, nh, kd); v, dout, dv (B, N, nh, hd)
// ---------------------------------------------------------------------------------------------------------------
constexpr int AT_THREADS = 128;

// pass A, per query row i: D_i = sum_j p_ij dP_ij, dS_ij = p_ij (dP_ij - D_i), dQ_i = scale sum_j dS_ij k_j
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
  // D: warp butterflies, then the warp partials in a fixed order
  for (int o = 16; o; o >>= 1) dsum += __shfl_xor_sync(0xffffffffu, dsum, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = dsum;
  __syncthreads();
  float D = red[0];
  for (int w = 1; w < AT_THREADS / 32; w++) D += red[w];
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

// pass B, per key row j: dV_j = sum_i p_ij dO_i, dK_j = scale sum_i dS_ij q_i
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
// Register-blocked backward for kd = 32, hd = 64 (every YOLOv11 size; N <= 448 tokens), same blocking as
// attention_tiled_32x64_kernel: 16-byte shared-memory reads, two rows per warp sharing every operand, global fills as
// batches of independent vector loads.  Row strides 36 (K / Q) and 68 (V / dO) floats keep
// both "a lane owns a row" (LDS.128 along the row) and "a lane owns a channel" (scalar / LDS.64 down a column) reads
// bank-conflict free.  D_i = sum_d dO_id O_id (= sum_j P_ij dP_ij) comes from the recomputed forward output.
// ---------------------------------------------------------------------------------------------------------------
constexpr int AB_T = 16, AB_THREADS = 256, AB_LDK = 36, AB_LDV = 68;
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

int attention_backward_f32(const float* q, const float* k, const float* v, const float* dout, int B, int N, int nh, int kd,
                           int hd, float scale, float* dq, float* dk, float* dv, cudaStream_t s) {
  if (int rc = attention_check(B, N, nh, kd, hd)) return rc;
  float* stats = nullptr;  // row max | row sum | row D, each (B, nh, N)
  const size_t n = (size_t)B * nh * N;
  YB_CUDA_CHECK(cudaMallocAsync((void**)&stats, (3 * n + (size_t)B * N * nh * hd) * sizeof(float), s));
  float* tmp_out = stats + 3 * n;  // the forward output is recomputed only for its row statistics
  int rc = attention_forward_f32(q, k, v, B, N, nh, kd, hd, scale, tmp_out, stats, stats + n, s);
  cudaError_t ce = cudaSuccess;
  if (!rc && kd == 32 && hd == 64 && ab_fits(N)) {
    ce = smem_limit((const void*)attn_bwd_q_32x64, ab_smem_bytes(N, 0), false);
    if (ce == cudaSuccess) ce = smem_limit((const void*)attn_bwd_kv_32x64, ab_smem_bytes(N, 1), false);
    if (ce == cudaSuccess) {
      const dim3 grid((N + AB_T - 1) / AB_T, nh, B);
      attn_bwd_q_32x64<<<grid, AB_THREADS, ab_smem_bytes(N, 0), s>>>(q, k, v, dout, tmp_out, stats, stats + n, stats + 2 * n, dq, N, nh, scale);
      attn_bwd_kv_32x64<<<grid, AB_THREADS, ab_smem_bytes(N, 1), s>>>(q, k, v, dout, stats, stats + n, stats + 2 * n, dk, dv, N, nh, scale);
      ce = cudaGetLastError();
    }
  } else if (!rc) {  // shared memory: N + kd + hd (q pass) and 2 N + kd + hd (kv pass) floats, within attention_check's limit
    const size_t smem_q = ((size_t)N + kd + hd) * sizeof(float), smem_kv = ((size_t)2 * N + kd + hd) * sizeof(float);
    ce = smem_limit((const void*)attn_backward_q_kernel, smem_q, false);
    if (ce == cudaSuccess) ce = smem_limit((const void*)attn_backward_kv_kernel, smem_kv, false);
    if (ce == cudaSuccess) {
      attn_backward_q_kernel<<<dim3(N, nh, B), AT_THREADS, smem_q, s>>>(q, k, v, dout, stats, stats + n, stats + 2 * n, dq, N, nh, kd,
                                                                         hd, scale);
      attn_backward_kv_kernel<<<dim3(N, nh, B), AT_THREADS, smem_kv, s>>>(q, k, v, dout, stats, stats + n, stats + 2 * n, dk, dv, N,
                                                                           nh, kd, hd, scale);
      ce = cudaGetLastError();
    }
  }
  if (ce != cudaSuccess) { set_error("attention backward launch failed"); rc = YB_ERR_CUDA; }
  cudaFreeAsync(stats, s);
  return rc;
}

}  // namespace yb

using namespace yb;

extern "C" {
int32_t yb_attention_forward_f32(const float* q, const float* k, const float* v, int32_t batch, int32_t tokens, int32_t heads,
                                 int32_t key_dim, int32_t head_dim, float scale, float* out, void* stream) {
  if (!q || !k || !v || !out) { set_error("yb_attention_forward_f32: null argument"); return YB_ERR_INVALID_ARG; }
  if (!have_device("yb_attention_forward_f32")) return YB_ERR_NO_DEVICE;
  return attention_forward_f32(q, k, v, batch, tokens, heads, key_dim, head_dim, scale, out, nullptr, nullptr, (cudaStream_t)stream);
}

int32_t yb_attention_backward_f32(const float* q, const float* k, const float* v, const float* dout, int32_t batch, int32_t tokens,
                                  int32_t heads, int32_t key_dim, int32_t head_dim, float scale, float* dq, float* dk, float* dv,
                                  void* stream) {
  if (!q || !k || !v || !dout || !dq || !dk || !dv) { set_error("yb_attention_backward_f32: null argument"); return YB_ERR_INVALID_ARG; }
  if (!have_device("yb_attention_backward_f32")) return YB_ERR_NO_DEVICE;
  return attention_backward_f32(q, k, v, dout, batch, tokens, heads, key_dim, head_dim, scale, dq, dk, dv, (cudaStream_t)stream);
}

}  // extern "C"
