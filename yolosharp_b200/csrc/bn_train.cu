// Train-mode BatchNorm2d + SiLU of the reference's Conv block (Modules/Convs.cs:36-56 with `yolo.train()`,
// YoloBaseTaskModel.cs:299,325): forward with batch statistics + running-statistics update, and backward.
//
//   forward   z (M = B*H*W rows, C channels, NHWC fp32) -> mean_c, var_c over the M rows (biased, two-pass),
//             y = SiLU(gamma * (z - mean) * invstd + beta), invstd = 1/sqrt(var + eps);
//             running_mean = (1-m) running_mean + m mean, running_var = (1-m) running_var + m var * M/(M-1)
//             (PyTorch BatchNorm2d semantics; the reference builds BatchNorm2d(eps 1e-3, momentum 0.03))
//   backward  u = gamma * xhat + beta, g = dy * SiLU'(u);  dbeta = sum g, dgamma = sum g*xhat,
//             dz = gamma * invstd * (g - dbeta/M - xhat * dgamma/M)
//
// All three passes are column reductions over a tall NHWC matrix: every block owns 32 channels x a slab of rows
// (32 x 8 threads, 128-byte coalesced rows), writes one partial per (slab, channel), and a second tiny kernel folds
// the partials in a fixed order - deterministic, no atomics.  HBM-bound: forward reads z twice (+1 in the
// elementwise pass) and writes y once; backward reads z, dy twice and writes dz.
#include <algorithm>

#include "common.cuh"

namespace yb {

namespace {

constexpr int BN_TX = 32, BN_TY = 8, BN_ROWS_PER_BLOCK = 256, BN_MAX_SLABS = 512;
// rows per slab: 256, or more for tall matrices so that the serial fold of the per-slab partials (bn_finish_kernel, one
// thread per channel) stays <= 512 steps (the 1.6 M-row first layers would otherwise have 6 400 slabs)
static int bn_rows_per_block(long long M) {
  const long long r = (M + BN_MAX_SLABS - 1) / BN_MAX_SLABS;
  return (int)std::max<long long>(BN_ROWS_PER_BLOCK, (r + BN_TY - 1) / BN_TY * BN_TY);
}

__device__ __forceinline__ float silu_grad(float u) {
  const float s = 1.f / (1.f + expf(-u));
  return s * (1.f + u * (1.f - s));
}

// mode 0: sum z                      -> p0
// mode 1: sum (z - mean)^2           -> p0
// mode 2: sum g, sum g * xhat        -> p0, p1   (g = dy * SiLU'(gamma*xhat+beta))
// mode 3: sum (z - K), sum (z - K)^2 -> p0, p1   one pass over z for mean AND variance; K = z[row 0][c] is a shift close to
//         the mean (a sample of the channel), so var = (S2 - S1^2 / M) / M cancels at most a few bits
//         (relative error ~ eps * (1 + (K - mean)^2 / var)); the two-pass modes 0 / 1 read every activation twice
__global__ void __launch_bounds__(BN_TX* BN_TY) bn_partial_kernel(int mode, int act, const float* __restrict__ z, const float* __restrict__ dy,
                                                                long long M, int C, int pitch, int dpitch,
                                                                const float* __restrict__ mean, const float* __restrict__ invstd,
                                                                const float* __restrict__ gamma, const float* __restrict__ beta,
                                                                float* __restrict__ p0, float* __restrict__ p1, int rpb) {
  const int c = blockIdx.x * BN_TX + threadIdx.x;
  const long long r0 = (long long)blockIdx.y * rpb;
  float a0 = 0.f, a1 = 0.f;
  if (c < C) {
    const float mu = mode == 3 ? z[c] : (mode ? mean[c] : 0.f);
    const float is = mode == 2 ? invstd[c] : 0.f, ga = mode == 2 ? gamma[c] : 0.f, be = mode == 2 ? beta[c] : 0.f;
    for (long long r = r0 + threadIdx.y; r < min(M, r0 + rpb); r += BN_TY) {
      const float v = z[r * pitch + c];
      if (mode == 0) {
        a0 += v;
      } else if (mode == 1) {
        const float d = v - mu;
        a0 += d * d;
      } else if (mode == 3) {
        const float d = v - mu;
        a0 += d;
        a1 = fmaf(d, d, a1);
      } else {
        const float xh = (v - mu) * is;
        const float g = dy[r * dpitch + c] * (act ? silu_grad(ga * xh + be) : 1.f);
        a0 += g;
        a1 += g * xh;
      }
    }
  }
  __shared__ float s0[BN_TY][BN_TX], s1[BN_TY][BN_TX];
  s0[threadIdx.y][threadIdx.x] = a0;
  s1[threadIdx.y][threadIdx.x] = a1;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    float t0 = 0.f, t1 = 0.f;
    for (int k = 0; k < BN_TY; k++) { t0 += s0[k][threadIdx.x]; t1 += s1[k][threadIdx.x]; }
    p0[(size_t)blockIdx.y * C + c] = t0;
    if (mode >= 2) p1[(size_t)blockIdx.y * C + c] = t1;
  }
}

// (The kernel is bound by rows in flight, not by load width.)
// fold the per-slab partials in a FIXED order; step 0 -> mean, step 1 -> var / invstd / running stats, step 2 -> dgamma,
// dbeta, step 3 -> mean / var from shifted sums.  Block = 32 channels x 8 lanes: lane y sums slabs y, y+8, ... in order,
// the 8 partial sums are then added in lane order (one thread per channel walking 512 slabs serially would be a long
// dependent-load chain).
__global__ void __launch_bounds__(256) bn_finish_kernel(int step, const float* __restrict__ p0, const float* __restrict__ p1, int slabs, int C,
                                 long long M, float eps, float momentum, float* __restrict__ mean, float* __restrict__ invstd,
                                 float* __restrict__ running_mean, float* __restrict__ running_var, float* __restrict__ dgamma,
                                 float* __restrict__ dbeta) {
  const int c = blockIdx.x * 32 + threadIdx.x;
  __shared__ float f0[8][32], f1[8][32];
  float a0 = 0.f, a1 = 0.f;
  if (c < C)
    for (int s = threadIdx.y; s < slabs; s += 8) {
      a0 += p0[(size_t)s * C + c];
      if (step >= 2) a1 += p1[(size_t)s * C + c];
    }
  f0[threadIdx.y][threadIdx.x] = a0;
  f1[threadIdx.y][threadIdx.x] = a1;
  __syncthreads();
  if (threadIdx.y != 0 || c >= C) return;
  float t0 = 0.f, t1 = 0.f;
  for (int k = 0; k < 8; k++) { t0 += f0[k][threadIdx.x]; t1 += f1[k][threadIdx.x]; }
  if (step == 3) {  // shifted sums (mode 3): running_mean carries the shift pointer's value z[0][c] via `dgamma`
    const float K = dgamma[c];
    const float d = t0 / (float)M;
    const float mu = K + d;
    const float var = fmaxf(t1 / (float)M - d * d, 0.f);  // biased: used for normalisation
    mean[c] = mu;
    invstd[c] = 1.f / sqrtf(var + eps);
    if (running_mean) {
      const float unbiased = M > 1 ? var * ((float)M / (float)(M - 1)) : var;
      running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mu;
      running_var[c] = (1.f - momentum) * running_var[c] + momentum * unbiased;
    }
  } else if (step == 0) {
    mean[c] = t0 / (float)M;
  } else if (step == 1) {
    const float var = t0 / (float)M;  // biased: used for normalisation
    invstd[c] = 1.f / sqrtf(var + eps);
    if (running_mean) {
      const float unbiased = M > 1 ? t0 / (float)(M - 1) : var;
      running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mean[c];
      running_var[c] = (1.f - momentum) * running_var[c] + momentum * unbiased;
    }
  } else {
    dbeta[c] = t0;
    dgamma[c] = t1;
  }
}

// ---- vectorised statistics pass with the fold fused in -----------------------------------------------------------------
// C % 4 == 0: a thread owns 4 adjacent channels (16-byte loads) and walks its slab's rows 4 at a time, all loads of a batch
// issued before the first add (the scalar kernel above keeps one 4-byte load per thread in flight and reaches a third of the
// HBM rate on the 1.6 M-row layers).  Block = LX channel lanes x LY rows (LX * LY = 256).  Sums are taken in row order per
// thread, folded over LY in lane order, written per slab; the block that arrives LAST on its channel column (a ticket from
// `counter`) folds the slabs in slab order and finishes the statistics - same fixed summation order whichever block it is,
// so the result is deterministic, and the 162 bn_finish launches of a YOLOv11s step disappear.
struct BnStat {
  const float *z, *dy;
  long long M;
  int C, pitch, dpitch, rpb, slabs, act;
  const float *mean, *invstd, *gamma, *beta;
  float *p0, *p1;
  unsigned* counter;  // one per channel column, zero on entry, left zero
  float eps, momentum;
  float *o_mean, *o_invstd, *running_mean, *running_var, *dgamma, *dbeta;
};

// rows per batch: 8 x 16 B (forward, z only) / 2 x 2 x 16 B (backward, z and dy) in flight per thread.  The backward pass
// is instruction-bound (SiLU' = exp + two divisions per element), so occupancy matters more than loads in flight: a batch
// of 2 fits 64 registers = 4 CTAs per SM
constexpr int BN4_U_FWD = 8, BN4_U_BWD = 2;

template <int MODE>  // 3: forward shifted sums (S1, S2 about K = z[row 0]); 2: backward sums (sum g, sum g * xhat)
__global__ void __launch_bounds__(256, 4) bn_stats4_kernel(const BnStat a) {
  pdl_wait();
  pdl_trigger();
  const int LX = blockDim.x, LY = blockDim.y, tx = threadIdx.x, ty = threadIdx.y;
  const int c = (blockIdx.x * LX + tx) * 4;
  const bool on = c < a.C;
  __shared__ float red[8][256];
  __shared__ int s_last;
  constexpr int BN4_U = MODE == 3 ? BN4_U_FWD : BN4_U_BWD;
  float s0[4] = {0.f, 0.f, 0.f, 0.f}, s1[4] = {0.f, 0.f, 0.f, 0.f};
  float4 K = make_float4(0.f, 0.f, 0.f, 0.f), IS = K, GA = K, BE = K;
  if (on) {
    if (MODE == 3) {
      K = *reinterpret_cast<const float4*>(a.z + c);
    } else {
      // per-channel vectors may sit at any 4-byte offset of the caller's flat buffers: scalar loads
      K = make_float4(a.mean[c], a.mean[c + 1], a.mean[c + 2], a.mean[c + 3]);
      IS = make_float4(a.invstd[c], a.invstd[c + 1], a.invstd[c + 2], a.invstd[c + 3]);
      GA = make_float4(a.gamma[c], a.gamma[c + 1], a.gamma[c + 2], a.gamma[c + 3]);
      BE = make_float4(a.beta[c], a.beta[c + 1], a.beta[c + 2], a.beta[c + 3]);
    }
    const long long r0 = (long long)blockIdx.y * a.rpb, r1 = min(a.M, r0 + a.rpb);
    const float kk[4] = {K.x, K.y, K.z, K.w}, ii[4] = {IS.x, IS.y, IS.z, IS.w};
    const float gg[4] = {GA.x, GA.y, GA.z, GA.w}, bb[4] = {BE.x, BE.y, BE.z, BE.w};
    auto acc = [&](const float4& v, const float4& d) {
      const float vv[4] = {v.x, v.y, v.z, v.w}, dd[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
      for (int j = 0; j < 4; j++) {
        if (MODE == 3) {
          const float e = vv[j] - kk[j];
          s0[j] += e;
          s1[j] = fmaf(e, e, s1[j]);
        } else {
          const float xh = (vv[j] - kk[j]) * ii[j];
          const float g = dd[j] * (a.act ? silu_grad(gg[j] * xh + bb[j]) : 1.f);
          s0[j] += g;
          s1[j] += g * xh;
        }
      }
    };
    // this thread's rows: r0 + ty, + LY, ...; full batches of BN4_U rows with every load issued before the first add
    // (plain pointer steps and an int trip count: with 64-bit row indices or a guarded load per row the compiler keeps a
    // single load in flight)
    const long long span = r1 - r0 - ty;
    const int nrows = span > 0 ? (int)((span + LY - 1) / LY) : 0;
    const float* zp = a.z + (r0 + ty) * a.pitch + c;
    const float* dp = MODE == 2 ? a.dy + (r0 + ty) * a.dpitch + c : nullptr;
    const size_t zs = (size_t)LY * a.pitch, ds = MODE == 2 ? (size_t)LY * a.dpitch : 0;
    int it = 0;
#pragma unroll 1
    for (; it + BN4_U <= nrows; it += BN4_U) {
      float4 v[BN4_U], d[BN4_U];
#pragma unroll
      for (int u = 0; u < BN4_U; u++) {
        v[u] = __ldg(reinterpret_cast<const float4*>(zp + u * zs));
        if (MODE == 2) d[u] = __ldg(reinterpret_cast<const float4*>(dp + u * ds));
        else d[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      zp += BN4_U * zs;
      if (MODE == 2) dp += BN4_U * ds;
#pragma unroll
      for (int u = 0; u < BN4_U; u++) acc(v[u], d[u]);
    }
#pragma unroll 1
    for (; it < nrows; it++) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(zp));
      const float4 d = MODE == 2 ? __ldg(reinterpret_cast<const float4*>(dp)) : make_float4(0.f, 0.f, 0.f, 0.f);
      zp += zs;
      if (MODE == 2) dp += ds;
      acc(v, d);
    }
  }
  const int t = ty * LX + tx;
#pragma unroll
  for (int j = 0; j < 4; j++) { red[j][t] = s0[j]; red[4 + j][t] = s1[j]; }
  __syncthreads();
  // fold over the LY row lanes in lane order: thread (x, j) -> channel lane x, component j of (s0[0..3], s1[0..3])
  if (t < LX * 8) {
    const int j = t / LX, x = t - j * LX;
    float f = 0.f;
    for (int y = 0; y < LY; y++) f += red[j][y * LX + x];
    const int ch = (blockIdx.x * LX + x) * 4 + (j & 3);
    if (ch < a.C) (j < 4 ? a.p0 : a.p1)[(size_t)blockIdx.y * a.C + ch] = f;
  }
  __threadfence();
  __syncthreads();
  if (t == 0) s_last = atomicAdd(&a.counter[blockIdx.x], 1u) == (unsigned)(a.slabs - 1);
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // the last block of this channel column: fold the slabs (lane y takes slabs y, y + LY, ... in order; lanes added in order)
  float4 q0 = make_float4(0.f, 0.f, 0.f, 0.f), q1 = q0;
  if (on) {
    // 4 slabs per batch, loads first (a one-load-at-a-time walk over 100 slabs per lane pays the L2 latency 100 times)
    const int mine = a.slabs > ty ? (a.slabs - ty + LY - 1) / LY : 0;
    const float* f0 = a.p0 + (size_t)ty * a.C + c;
    const float* f1 = a.p1 + (size_t)ty * a.C + c;
    const size_t fs = (size_t)LY * a.C;
    int k = 0;
#pragma unroll 1
    for (; k + 4 <= mine; k += 4) {
      float4 u0[4], u1[4];
#pragma unroll
      for (int u = 0; u < 4; u++) {
        u0[u] = __ldcg(reinterpret_cast<const float4*>(f0 + u * fs));
        u1[u] = __ldcg(reinterpret_cast<const float4*>(f1 + u * fs));
      }
      f0 += 4 * fs;
      f1 += 4 * fs;
#pragma unroll
      for (int u = 0; u < 4; u++) {
        q0.x += u0[u].x; q0.y += u0[u].y; q0.z += u0[u].z; q0.w += u0[u].w;
        q1.x += u1[u].x; q1.y += u1[u].y; q1.z += u1[u].z; q1.w += u1[u].w;
      }
    }
#pragma unroll 1
    for (; k < mine; k++) {
      const float4 u0 = __ldcg(reinterpret_cast<const float4*>(f0));
      const float4 u1 = __ldcg(reinterpret_cast<const float4*>(f1));
      f0 += fs;
      f1 += fs;
      q0.x += u0.x; q0.y += u0.y; q0.z += u0.z; q0.w += u0.w;
      q1.x += u1.x; q1.y += u1.y; q1.z += u1.z; q1.w += u1.w;
    }
  }
  __syncthreads();
  red[0][t] = q0.x; red[1][t] = q0.y; red[2][t] = q0.z; red[3][t] = q0.w;
  red[4][t] = q1.x; red[5][t] = q1.y; red[6][t] = q1.z; red[7][t] = q1.w;
  __syncthreads();
  if (t == 0) a.counter[blockIdx.x] = 0;
  if (t >= LX * 4) return;
  const int j = t / LX, x = t - j * LX;
  const int ch = (blockIdx.x * LX + x) * 4 + j;
  if (ch >= a.C) return;
  float t0 = 0.f, t1 = 0.f;
  for (int y = 0; y < LY; y++) { t0 += red[j][y * LX + x]; t1 += red[4 + j][y * LX + x]; }
  if (MODE == 3) {
    const float Kc = a.z[ch];
    const float dm = t0 / (float)a.M;
    const float mu = Kc + dm;
    const float var = fmaxf(t1 / (float)a.M - dm * dm, 0.f);  // biased: used for normalisation
    a.o_mean[ch] = mu;
    a.o_invstd[ch] = 1.f / sqrtf(var + a.eps);
    if (a.running_mean) {
      const float unbiased = a.M > 1 ? var * ((float)a.M / (float)(a.M - 1)) : var;
      a.running_mean[ch] = (1.f - a.momentum) * a.running_mean[ch] + a.momentum * mu;
      a.running_var[ch] = (1.f - a.momentum) * a.running_var[ch] + a.momentum * unbiased;
    }
  } else {
    a.dbeta[ch] = t0;
    a.dgamma[ch] = t1;
  }
}

// launch geometry of the vectorised pass: LX channel lanes (power of two <= 32), slabs sized for ~4 blocks per SM
struct Bn4Plan { int LX, LY, colblocks, rpb, slabs; };
static Bn4Plan bn4_plan(long long M, int C, int U) {
  Bn4Plan p;
  const int c4 = C / 4;
  p.LX = 1;
  while (p.LX < c4 && p.LX < 32) p.LX <<= 1;
  p.LY = 256 / p.LX;
  p.colblocks = (c4 + p.LX - 1) / p.LX;
  const int want = std::min(BN_MAX_SLABS, std::max(1, 592 / p.colblocks));
  const long long step = (long long)p.LY * U;
  long long rpb = (M + want - 1) / want;
  rpb = std::max(step, (rpb + step - 1) / step * step);
  p.rpb = (int)rpb;
  p.slabs = (int)((M + rpb - 1) / rpb);
  return p;
}
static bool bn4_ok(long long M, int C, const void* z, int pitch, const void* dy, int dpitch) {
  return C % 4 == 0 && pitch % 4 == 0 && dpitch % 4 == 0 && (uintptr_t)z % 16 == 0 && (uintptr_t)dy % 16 == 0 && M * C / 4 < (1ll << 31);
}

__global__ void bn_silu_apply_kernel(const float* __restrict__ z, long long M, int C, int pitch, int opitch,
                                     const float* __restrict__ mean, const float* __restrict__ invstd,
                                     const float* __restrict__ gamma, const float* __restrict__ beta, int act, float* __restrict__ y) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * C) return;
  const long long r = i / C;
  const int c = (int)(i - r * C);
  const float u = gamma[c] * (z[r * pitch + c] - mean[c]) * invstd[c] + beta[c];
  y[r * opitch + c] = act ? silu_f(u) : u;
}

__global__ void bn_silu_dz_kernel(const float* __restrict__ z, const float* __restrict__ dy, long long M, int C, int pitch, int dpitch,
                                  int opitch, const float* __restrict__ mean, const float* __restrict__ invstd,
                                  const float* __restrict__ gamma, const float* __restrict__ beta, int act,
                                  const float* __restrict__ dgamma, const float* __restrict__ dbeta, float* __restrict__ dz) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * C) return;
  const long long r = i / C;
  const int c = (int)(i - r * C);
  const float xh = (z[r * pitch + c] - mean[c]) * invstd[c];
  const float g = dy[r * dpitch + c] * (act ? silu_grad(gamma[c] * xh + beta[c]) : 1.f);
  const float inv_m = 1.f / (float)M;
  dz[r * opitch + c] = gamma[c] * invstd[c] * (g - dbeta[c] * inv_m - xh * dgamma[c] * inv_m);
}

// Elementwise passes, 4 channels per thread: a thread owns one channel quad and walks rows r0 + ty, + LY, ... of its slab, so
// the per-channel vectors (mean, invstd, gamma, beta [, dgamma, dbeta]) are loaded ONCE per thread instead of once per
// element and there is no index division.
struct BnRows {
  const float *z, *dy;
  float* out;
  long long M;
  int C, pitch, dpitch, opitch, rpb, act;
  const float *mean, *invstd, *gamma, *beta, *dgamma, *dbeta;
  float inv_m;
};

template <int BWD>  // 0: y = act(gamma * xhat + beta); 1: dz from dy (BatchNorm + SiLU backward)
__global__ void __launch_bounds__(256, BWD ? 3 : 4) bn_rows4_kernel(const BnRows a) {
  pdl_wait();
  pdl_trigger();
  const int LX = blockDim.x, LY = blockDim.y, ty = threadIdx.y;
  const int c = (blockIdx.x * LX + threadIdx.x) * 4;
  if (c >= a.C) return;
  float mu[4], is[4], ga[4], be[4], dg[4], db[4];
#pragma unroll
  for (int j = 0; j < 4; j++) {
    mu[j] = a.mean[c + j]; is[j] = a.invstd[c + j]; ga[j] = a.gamma[c + j]; be[j] = a.beta[c + j];
    dg[j] = BWD ? a.dgamma[c + j] : 0.f;
    db[j] = BWD ? a.dbeta[c + j] : 0.f;
  }
  const float inv_m = a.inv_m;
  auto fwd = [&](const float4& v) {
    float4 u;
    u.x = ga[0] * (v.x - mu[0]) * is[0] + be[0]; u.y = ga[1] * (v.y - mu[1]) * is[1] + be[1];
    u.z = ga[2] * (v.z - mu[2]) * is[2] + be[2]; u.w = ga[3] * (v.w - mu[3]) * is[3] + be[3];
    if (a.act) { u.x = silu_f(u.x); u.y = silu_f(u.y); u.z = silu_f(u.z); u.w = silu_f(u.w); }
    return u;
  };
  auto bwd = [&](const float4& v, const float4& d) {
    const float vv[4] = {v.x, v.y, v.z, v.w}, dd[4] = {d.x, d.y, d.z, d.w};
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const float xh = (vv[j] - mu[j]) * is[j];
      const float g = dd[j] * (a.act ? silu_grad(ga[j] * xh + be[j]) : 1.f);
      o[j] = ga[j] * is[j] * (g - db[j] * inv_m - xh * dg[j] * inv_m);
    }
    return make_float4(o[0], o[1], o[2], o[3]);
  };
  const long long r0 = (long long)blockIdx.y * a.rpb, r1 = min(a.M, r0 + a.rpb);
  const long long span = r1 - r0 - ty;
  const int nrows = span > 0 ? (int)((span + LY - 1) / LY) : 0;
  const float* zp = a.z + (r0 + ty) * a.pitch + c;
  const float* dp = BWD ? a.dy + (r0 + ty) * a.dpitch + c : nullptr;
  float* op = a.out + (r0 + ty) * a.opitch + c;
  const size_t zs = (size_t)LY * a.pitch, ds = BWD ? (size_t)LY * a.dpitch : 0, os = (size_t)LY * a.opitch;
  int it = 0;
#pragma unroll 1
  for (; it + 2 <= nrows; it += 2) {
    const float4 v0 = __ldg(reinterpret_cast<const float4*>(zp)), v1 = __ldg(reinterpret_cast<const float4*>(zp + zs));
    float4 o0, o1;
    if (BWD) {
      const float4 d0 = __ldg(reinterpret_cast<const float4*>(dp)), d1 = __ldg(reinterpret_cast<const float4*>(dp + ds));
      o0 = bwd(v0, d0);
      o1 = bwd(v1, d1);
      dp += 2 * ds;
    } else {
      o0 = fwd(v0);
      o1 = fwd(v1);
    }
    *reinterpret_cast<float4*>(op) = o0;
    *reinterpret_cast<float4*>(op + os) = o1;
    zp += 2 * zs;
    op += 2 * os;
  }
  if (it < nrows) {
    const float4 v0 = __ldg(reinterpret_cast<const float4*>(zp));
    *reinterpret_cast<float4*>(op) = BWD ? bwd(v0, __ldg(reinterpret_cast<const float4*>(dp))) : fwd(v0);
  }
}

struct BnRowsPlan { int LX, LY, colblocks, rpb, slabs; };
static BnRowsPlan bn_rows_plan(long long M, int C) {
  BnRowsPlan p;
  const int c4 = C / 4;
  p.LX = 1;
  while (p.LX < c4 && p.LX < 32) p.LX <<= 1;
  p.LY = 256 / p.LX;
  p.colblocks = (c4 + p.LX - 1) / p.LX;
  const long long want = std::max(1, 2368 / p.colblocks);  // ~16 CTAs per SM over the launch: 4 resident, 4 waves
  const long long step = (long long)p.LY * 2;
  long long rpb = (M + want - 1) / want;
  rpb = std::max(step, (rpb + step - 1) / step * step);
  p.rpb = (int)rpb;
  p.slabs = (int)((M + rpb - 1) / rpb);
  return p;
}

}  // namespace

int bn_silu_train_forward(const float* z, long long M, int C, int pitch, const float* gamma, const float* beta, float eps,
                          float momentum, int act, float* running_mean, float* running_var, float* y, int ypitch,
                          float* save_mean, float* save_invstd, cudaStream_t s, unsigned* counters) {
  if (M <= 0 || C <= 0 || pitch < C || ypitch < C) {
    set_error("yb_bn_silu_train_forward: bad shape");
    return YB_ERR_SHAPE;
  }
  float* part = nullptr;
  if (bn4_ok(M, C, z, pitch, z, pitch)) {
    // one vectorised pass over z, statistics finished by the last block of each channel column
    const Bn4Plan pl = bn4_plan(M, C, BN4_U_FWD);
    const size_t nf = (size_t)2 * pl.slabs * C;
    const bool own = !counters || pl.colblocks > 64;
    YB_CUDA_CHECK(cudaMallocAsync((void**)&part, nf * sizeof(float) + pl.colblocks * sizeof(unsigned), s));
    if (own) YB_CUDA_CHECK(cudaMemsetAsync(part + nf, 0, pl.colblocks * sizeof(unsigned), s));
    BnStat a{};
    a.z = z; a.M = M; a.C = C; a.pitch = pitch; a.rpb = pl.rpb; a.slabs = pl.slabs; a.act = act;
    a.p0 = part; a.p1 = part + (size_t)pl.slabs * C; a.counter = own ? reinterpret_cast<unsigned*>(part + nf) : counters;
    a.eps = eps; a.momentum = momentum; a.o_mean = save_mean; a.o_invstd = save_invstd;
    a.running_mean = running_mean; a.running_var = running_var;
    YB_CUDA_CHECK(launch_pdl(bn_stats4_kernel<3>, dim3(pl.colblocks, pl.slabs), dim3(pl.LX, pl.LY), 0, s, a));
  } else {
    const int rpb = bn_rows_per_block(M);
    const int slabs = (int)((M + rpb - 1) / rpb);
    YB_CUDA_CHECK(cudaMallocAsync((void**)&part, (size_t)2 * slabs * C * sizeof(float), s));
    const dim3 grid((C + BN_TX - 1) / BN_TX, slabs), block(BN_TX, BN_TY);
    const dim3 fb(32, 8);
    const int fg = (C + 31) / 32;
    // one pass over z: per-slab sums of (z - K) and (z - K)^2 about the shift K = z[row 0], folded in slab order
    bn_partial_kernel<<<grid, block, 0, s>>>(3, act, z, nullptr, M, C, pitch, 0, nullptr, nullptr, nullptr, nullptr, part,
                                            part + (size_t)slabs * C, rpb);
    bn_finish_kernel<<<fg, fb, 0, s>>>(3, part, part + (size_t)slabs * C, slabs, C, M, eps, momentum, save_mean, save_invstd, running_mean,
                                       running_var, const_cast<float*>(z) /* the shift row, read only */, nullptr);
  }
  if (int rc = bn_silu_apply(z, M, C, pitch, save_mean, save_invstd, gamma, beta, act, y, ypitch, s)) return rc;
  YB_CUDA_CHECK(cudaFreeAsync(part, s));
  return YB_OK;
}

int bn_silu_apply(const float* z, long long M, int C, int pitch, const float* mean, const float* invstd, const float* gamma,
                  const float* beta, int act, float* y, int ypitch, cudaStream_t s) {
  const long long total = M * C;
  if (C % 4 == 0 && pitch % 4 == 0 && ypitch % 4 == 0 && ((uintptr_t)z % 16 == 0) && ((uintptr_t)y % 16 == 0)) {
    const BnRowsPlan pl = bn_rows_plan(M, C);
    BnRows a{};
    a.z = z; a.out = y; a.M = M; a.C = C; a.pitch = pitch; a.opitch = ypitch; a.rpb = pl.rpb; a.act = act;
    a.mean = mean; a.invstd = invstd; a.gamma = gamma; a.beta = beta;
    YB_CUDA_CHECK(launch_pdl(bn_rows4_kernel<0>, dim3(pl.colblocks, pl.slabs), dim3(pl.LX, pl.LY), 0, s, a));
  } else {
    bn_silu_apply_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(z, M, C, pitch, ypitch, mean, invstd, gamma, beta, act, y);
  }
  YB_CUDA_CHECK(cudaGetLastError());
  return YB_OK;
}

int bn_silu_backward(const float* z, const float* dy, long long M, int C, int pitch, int dpitch, const float* gamma,
                     const float* beta, const float* save_mean, const float* save_invstd, int act, float* dz, int zpitch,
                     float* dgamma, float* dbeta, cudaStream_t s, unsigned* counters) {
  if (M <= 0 || C <= 0 || pitch < C || dpitch < C || zpitch < C) {
    set_error("yb_bn_silu_backward: bad shape");
    return YB_ERR_SHAPE;
  }
  float* part = nullptr;
  if (bn4_ok(M, C, z, pitch, dy, dpitch)) {
    const Bn4Plan pl = bn4_plan(M, C, BN4_U_BWD);
    const size_t nf = (size_t)2 * pl.slabs * C;
    const bool own = !counters || pl.colblocks > 64;
    YB_CUDA_CHECK(cudaMallocAsync((void**)&part, nf * sizeof(float) + pl.colblocks * sizeof(unsigned), s));
    if (own) YB_CUDA_CHECK(cudaMemsetAsync(part + nf, 0, pl.colblocks * sizeof(unsigned), s));
    BnStat a{};
    a.z = z; a.dy = dy; a.M = M; a.C = C; a.pitch = pitch; a.dpitch = dpitch; a.rpb = pl.rpb; a.slabs = pl.slabs; a.act = act;
    a.mean = save_mean; a.invstd = save_invstd; a.gamma = gamma; a.beta = beta;
    a.p0 = part; a.p1 = part + (size_t)pl.slabs * C; a.counter = own ? reinterpret_cast<unsigned*>(part + nf) : counters;
    a.dgamma = dgamma; a.dbeta = dbeta;
    YB_CUDA_CHECK(launch_pdl(bn_stats4_kernel<2>, dim3(pl.colblocks, pl.slabs), dim3(pl.LX, pl.LY), 0, s, a));
  } else {
    const int rpb = bn_rows_per_block(M);
    const int slabs = (int)((M + rpb - 1) / rpb);
    YB_CUDA_CHECK(cudaMallocAsync((void**)&part, (size_t)2 * slabs * C * sizeof(float), s));
    const dim3 grid((C + BN_TX - 1) / BN_TX, slabs), block(BN_TX, BN_TY);
    bn_partial_kernel<<<grid, block, 0, s>>>(2, act, z, dy, M, C, pitch, dpitch, save_mean, save_invstd, gamma, beta, part,
                                            part + (size_t)slabs * C, rpb);
    bn_finish_kernel<<<(C + 31) / 32, dim3(32, 8), 0, s>>>(2, part, part + (size_t)slabs * C, slabs, C, M, 0.f, 0.f, nullptr, nullptr, nullptr,
                                                     nullptr, dgamma, dbeta);
  }
  const long long total = M * C;
  if (C % 4 == 0 && pitch % 4 == 0 && dpitch % 4 == 0 && zpitch % 4 == 0 && ((uintptr_t)z % 16 == 0) && ((uintptr_t)dy % 16 == 0) &&
      ((uintptr_t)dz % 16 == 0)) {
    const BnRowsPlan pl = bn_rows_plan(M, C);
    BnRows a{};
    a.z = z; a.dy = dy; a.out = dz; a.M = M; a.C = C; a.pitch = pitch; a.dpitch = dpitch; a.opitch = zpitch; a.rpb = pl.rpb; a.act = act;
    a.mean = save_mean; a.invstd = save_invstd; a.gamma = gamma; a.beta = beta; a.dgamma = dgamma; a.dbeta = dbeta;
    a.inv_m = 1.f / (float)M;
    YB_CUDA_CHECK(launch_pdl(bn_rows4_kernel<1>, dim3(pl.colblocks, pl.slabs), dim3(pl.LX, pl.LY), 0, s, a));
  } else {
    bn_silu_dz_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(z, dy, M, C, pitch, dpitch, zpitch, save_mean, save_invstd, gamma, beta,
                                                                  act, dgamma, dbeta, dz);
  }
  YB_CUDA_CHECK(cudaGetLastError());
  YB_CUDA_CHECK(cudaFreeAsync(part, s));
  return YB_OK;
}

// AdamW step (torch.optim.AdamW semantics, the optimizer the reference builds in YoloBaseTaskModel.cs:142-160):
//   p *= 1 - lr*wd;  m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;  p -= lr/(1-b1^t) * m / (sqrt(v)/sqrt(1-b2^t) + eps)
__global__ void adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                             long long n, float lr, float b1, float b2, float eps, float wd, float bc1, float bc2_sqrt) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float gi = g[i];
  float pi = p[i] * (1.f - lr * wd);
  const float mi = b1 * m[i] + (1.f - b1) * gi;
  const float vi = b2 * v[i] + (1.f - b2) * gi * gi;
  m[i] = mi;
  v[i] = vi;
  const float denom = sqrtf(vi) / bc2_sqrt + eps;
  p[i] = pi - (lr / bc1) * (mi / denom);
}

int adamw_step(float* p, const float* g, float* m, float* v, long long n, int step, float lr, float b1, float b2, float eps,
               float wd, cudaStream_t s) {
  if (n <= 0 || step < 1) {
    set_error("yb_adamw_step: need n > 0 and step >= 1");
    return YB_ERR_INVALID_ARG;
  }
  const float bc1 = 1.f - powf(b1, (float)step), bc2_sqrt = sqrtf(1.f - powf(b2, (float)step));
  adamw_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(p, g, m, v, n, lr, b1, b2, eps, wd, bc1, bc2_sqrt);
  YB_CUDA_CHECK(cudaGetLastError());
  return YB_OK;
}

}  // namespace yb

// ------------------------------------------------------------------------------------------
// Convolution backward, fp32 CUDA-core parity path (the training-side twin of conv_generic_kernel: correct and
// deterministic first; the tensor-core dgrad / wgrad kernels of the throughput path will be checked against it).
//   dz (N, Ho, Wo, Cout) NHWC, weights in the reference's checkpoint layout (Cout, Cin, k, k)
//   dgrad  dx[n,h,w,ci] = sum_{kh,kw,co} dz[n,(h+pad-kh)/s,(w+pad-kw)/s,co] * W[co,ci,kh,kw]   (only exact divisions)
//   wgrad  dW[co,ci,kh,kw] = sum_{n,ho,wo} dz[n,ho,wo,co] * x[n,ho*s+kh-pad,wo*s+kw-pad,ci]
// ------------------------------------------------------------------------------------------
namespace yb {

namespace {

__global__ void conv_dgrad_kernel(const float* __restrict__ dz, const float* __restrict__ w, int N, int H, int W, int Cin, int Ho,
                                  int Wo, int Cout, int k, int stride, int pad, float* __restrict__ dx) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)N * H * W * Cin;
  if (i >= total) return;
  const int ci = (int)(i % Cin);
  long long p = i / Cin;
  const int x = (int)(p % W);
  p /= W;
  const int y = (int)(p % H);
  const int n = (int)(p / H);
  float acc = 0.f;
  for (int kh = 0; kh < k; kh++) {
    const int hn = y + pad - kh;
    if (hn < 0 || hn % stride) continue;
    const int ho = hn / stride;
    if (ho >= Ho) continue;
    for (int kw = 0; kw < k; kw++) {
      const int wn = x + pad - kw;
      if (wn < 0 || wn % stride) continue;
      const int wo = wn / stride;
      if (wo >= Wo) continue;
      const float* dzp = dz + (((size_t)n * Ho + ho) * Wo + wo) * Cout;
      const float* wp = w + ((size_t)ci * k + kh) * k + kw;  // + co * Cin*k*k
      for (int co = 0; co < Cout; co++) acc = fmaf(dzp[co], wp[(size_t)co * Cin * k * k], acc);
    }
  }
  dx[i] = acc;
}

// one block per (co, tap, slab of output rows): threads over ci, serial over the slab's pixels; the per-slab
// partials are folded in slab order by conv_wgrad_reduce_kernel (deterministic sums, no atomics)
__global__ void __launch_bounds__(128) conv_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dz, int N, int H, int W,
                                                        int Cin, int Ho, int Wo, int Cout, int k, int stride, int pad,
                                                        int rows_per_slab, float* __restrict__ part) {
  const int tap = blockIdx.x, co = blockIdx.y, slab = blockIdx.z;
  const int kh = tap / k, kw = tap - kh * k;
  const int r0 = slab * rows_per_slab, r1 = min(N * Ho, r0 + rows_per_slab);  // rows of the flattened (n, ho) index
  const size_t dw_size = (size_t)Cout * Cin * k * k;
  for (int ci = threadIdx.x; ci < Cin; ci += blockDim.x) {
    float acc = 0.f;
    for (int r = r0; r < r1; r++) {
      const int n = r / Ho, ho = r - n * Ho;
      const int hi = ho * stride + kh - pad;
      if (hi < 0 || hi >= H) continue;
      for (int wo = 0; wo < Wo; wo++) {
        const int wi = wo * stride + kw - pad;
        if (wi < 0 || wi >= W) continue;
        acc = fmaf(dz[(((size_t)n * Ho + ho) * Wo + wo) * Cout + co], x[(((size_t)n * H + hi) * W + wi) * Cin + ci], acc);
      }
    }
    part[(size_t)slab * dw_size + (((size_t)co * Cin + ci) * k + kh) * k + kw] = acc;
  }
}

__global__ void conv_wgrad_reduce_kernel(const float* __restrict__ part, int slabs, size_t dw_size, float* __restrict__ dw) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= dw_size) return;
  float t = 0.f;
  for (int s = 0; s < slabs; s++) t += part[(size_t)s * dw_size + i];
  dw[i] = t;
}

}  // namespace

int conv_backward_data(const float* dz, const float* w, int N, int H, int W, int Cin, int Cout, int k, int stride, int pad,
                       float* dx, cudaStream_t s) {
  if (N <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0 || k <= 0 || stride <= 0 || pad < 0) {
    set_error("yb_conv_backward_data: bad shape");
    return YB_ERR_SHAPE;
  }
  const int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
  const long long total = (long long)N * H * W * Cin;
  conv_dgrad_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(dz, w, N, H, W, Cin, Ho, Wo, Cout, k, stride, pad, dx);
  YB_CUDA_CHECK(cudaGetLastError());
  return YB_OK;
}

int conv_backward_weight(const float* x, const float* dz, int N, int H, int W, int Cin, int Cout, int k, int stride, int pad,
                         float* dw, cudaStream_t s) {
  if (N <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0 || k <= 0 || stride <= 0 || pad < 0) {
    set_error("yb_conv_backward_weight: bad shape");
    return YB_ERR_SHAPE;
  }
  const int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
  const size_t dw_size = (size_t)Cout * Cin * k * k;
  // enough slabs to fill the machine on the high-resolution layers, bounded partial buffer (<= 64 MB)
  int slabs = std::max(1, std::min(64, (N * Ho * Wo) / 2048));
  slabs = (int)std::max<size_t>(1, std::min<size_t>((size_t)slabs, ((size_t)16 << 20) / dw_size));
  slabs = std::min(slabs, N * Ho);
  const int rows_per_slab = (N * Ho + slabs - 1) / slabs;
  slabs = (N * Ho + rows_per_slab - 1) / rows_per_slab;
  float* part = nullptr;
  YB_CUDA_CHECK(cudaMallocAsync((void**)&part, (size_t)slabs * dw_size * sizeof(float), s));
  conv_wgrad_kernel<<<dim3(k * k, Cout, slabs), 128, 0, s>>>(x, dz, N, H, W, Cin, Ho, Wo, Cout, k, stride, pad, rows_per_slab, part);
  conv_wgrad_reduce_kernel<<<(unsigned)((dw_size + 255) / 256), 256, 0, s>>>(part, slabs, dw_size, dw);
  YB_CUDA_CHECK(cudaGetLastError());
  YB_CUDA_CHECK(cudaFreeAsync(part, s));
  return YB_OK;
}

}  // namespace yb
