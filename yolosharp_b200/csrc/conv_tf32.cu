// Tensor-core convolutions of the TRAINING step (fp32 storage, TF32 MMAs, fp32 accumulate in registers).
//
// Replaces, on the training path, what libtorch runs behind `Conv2d.forward` and `loss.backward()` for the Conv
// blocks of the reference (Modules/Convs.cs:44; Utils/Amp.cs:260-286 calls forward / backward / optimizer.step):
// forward, data gradient and weight gradient of a dense k x k convolution (k in {1, 3}, stride in {1, 2}), on the
// NHWC fp32 activations the training step keeps.  libtorch's own CUDA convolutions run TF32 tensor-core math by
// default (cudnn.allow_tf32), so TF32 products with fp32 accumulation are the reference's arithmetic class here;
// the fp32 CUDA-core kernels (yb_conv_forward_f32 / yb_conv_backward_*) stay as the parity twins these are tested
// against.
//
//   tf_conv_kernel   one implicit-GEMM kernel for forward AND data gradient.  M = 128 output positions (a BW x BH
//                    rectangle of one image, or 128 consecutive positions of the flattened batch for 1x1), N = output
//                    channels (tile <= 256), K = taps x input channels.  Both operands K-major: A = NHWC activations
//                    (one 4-D TMA box per tap and 32-channel slab, zero fill = padding, traversal stride = conv
//                    stride), B = weights re-packed per step as [tap][N][K] (3-D TMA box); wgmma m64nNk8 TF32 from
//                    two consumer warpgroups (64 rows each), one producer warp.  A launch is described
//                    by a TAP TABLE (box offset dh, dw + weight slab per tap), which covers
//                      forward          out(y,x) = sum_t in(y*s + kh - p, x*s + kw - p) W[kh][kw]
//                      dgrad, stride 1  dx(y,x)  = sum_t dz(y + p - kh, x + p - kw) W^T[kh][kw]
//                      dgrad, stride 2  four launches, one per output parity (py, px), each with the taps whose
//                                       (py + p - kh) and (px + p - kw) are even, writing every second position
//   tf_wgrad_kernel  dW[co][tap][ci] = sum_pixels dz[pix][co] * x[pix + tap][ci]: K = pixels, so both operands are
//                    MN-major - exactly the NHWC tiles TMA delivers (64 pixels x 32 channels, 128-byte SWIZZLE_128B
//                    rows).  wgmma reads TF32 operands K-major only, so eight warps run mma.sync m16n8k8 TF32 with
//                    fragments loaded from the swizzled tiles.  One CTA owns 128 output channels x (taps x 32 nb) input
//                    channels (<= 128 accumulator columns, 64 registers per thread), walks its share of the pixel tiles
//                    (split-K over pixels) and stores a partial; a fixed-order fold sums the partials into the
//                    checkpoint layout (deterministic, no atomics).
#include <cuda.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace yb {

constexpr int TF_MAX_STAGES = 8;
constexpr int TF_CONSUMER_WARPS = 8;                      // two warpgroups (tf_conv_kernel) / eight MMA warps (wgrad)
constexpr int TF_THREADS = 32 * TF_CONSUMER_WARPS + 32;  // + warp 8: TMA producer
// blocks of the stem wgrad: a fixed count, so that the partials and their fold order (and the result) do not depend on the GPU
constexpr int ST_WG_BLOCKS = 592;

// ------------------------------------------------------------------------------------------
// forward / data gradient
// ------------------------------------------------------------------------------------------
struct TfArgs {
  CUtensorMap tmA, tmB;
  TileGrid tg;
  float* out;
  const float* bias;                // [n_out] or nullptr (always set in the eval epilogue)
  const float* res;                 // eval epilogue: residual view added after the activation, or nullptr
  long long r_pitch;                // elements between consecutive output positions of `res`
  int act;                          // eval epilogue: 1 = SiLU after the bias
  long long o_img, o_row, o_pix;    // element strides of the output addressing
  long long o_off;
  int n_out;                        // valid output channels (columns >= n_out are not stored)
  int Ho, Wo;                       // extent of the output position grid the tiles cover
  int n_tile;
  int BW, BH;
  int in_stride;                    // A box origin = (w0 * in_stride + dw, h0 * in_stride + dh)
  int ntaps;
  int dh[9], dw[9], slab[9];
  int chunks, KK;                   // K slabs per tap, MMAs (K = 8) per slab
  int BK;
  int stages;
  uint32_t a_stride, b_stride, a_bytes, b_bytes;
  uint32_t layout, sbo16;  // wgmma layout type (1 = SWIZZLE_128B, 2 = 64B, 3 = 32B), 8-row group stride >> 4
};

template <int NT16, int KK>
__device__ __forceinline__ void tf_mainloop(const TfArgs& a, float* acc, uint32_t smemA, uint32_t smemB, uint32_t full0, uint32_t empty0,
                                            int& st, uint32_t& ph) {
  const uint32_t hi = wg_desc_hi(a.sbo16, a.layout);
  const uint32_t a_off = (threadIdx.x >> 7) * 8 * a.sbo16;  // warpgroup 1: rows 64.. = 8 groups of 8 rows further
  const bool leader = (threadIdx.x & 31) == 0;
  const int ksteps = a.ntaps * a.chunks;
  uint32_t pend = 0;  // slot read by the previous commit group
  for (int ks = 0; ks < ksteps; ks++) {
    mbar_wait(full0 + 8 * st, ph);
    const uint32_t a_lo = wg_desc_lo(smemA + st * a.a_stride) + a_off, b_lo = wg_desc_lo(smemB + st * a.b_stride);
    wg_fence();
#pragma unroll
    for (int k = 0; k < KK; k++)  // 8 fp32 = 32 bytes per K step inside the swizzled row
      wg_mma_n<NT16, true>(acc, a_lo + 2 * k, hi, b_lo + 2 * k, hi, KK * 2, (ks > 0 || k > 0) ? 1u : 0u);
    wg_commit();
    wg_wait<1>();
    __syncwarp();
    if (leader && pend) mbar_arrive(pend);
    pend = empty0 + 8 * st;
    ring_next(st, ph, a.stages);
  }
  wg_wait<0>();
  __syncwarp();
  if (leader && pend) mbar_arrive(pend);
  wg_fence_acc<NT16 * 8>(acc);
}

// EVAL = false: out = acc (+ bias), the training forward / dgrad.  EVAL = true: the eval-mode Conv block with BatchNorm
// folded into the weights and bias, out = [res +] act(acc + bias) (a template parameter, so that the training
// instantiations carry none of its registers)
template <int NT16, bool EVAL>
__global__ void __launch_bounds__(TF_THREADS, NT16 <= 4 ? 2 : 1) tf_conv_kernel(const __grid_constant__ TfArgs a) {
  // the barrier setup below overlaps the tail of the previous kernel (launch_pdl); pdl_wait() before any global access
  extern __shared__ __align__(1024) uint8_t tf_smem[];
  __shared__ __align__(8) uint64_t bars[2 * TF_MAX_STAGES];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t smem0 = (smem_u32(tf_smem) + 1023u) & ~1023u;
  const uint32_t smemA = smem0, smemB = smem0 + a.stages * a.a_stride;
  const uint32_t full0 = smem_u32(&bars[0]), empty0 = smem_u32(&bars[TF_MAX_STAGES]);
  if (threadIdx.x == 0) {
    for (int s = 0; s < a.stages; s++) { mbar_init(full0 + 8 * s, 1); mbar_init(empty0 + 8 * s, TF_CONSUMER_WARPS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();

  if (warp == TF_CONSUMER_WARPS) {
    if (lane == 0) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&a.tmA) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&a.tmB) : "memory");
      int st = 0;
      uint32_t ph = 0;
      for (int tile = blockIdx.x; tile < a.tg.total; tile += gridDim.x) {
        const TileCoord tc = tile_coord(a.tg, tile);
        const int wbase = tc.tw * a.BW * a.in_stride, hbase = tc.th * a.BH * a.in_stride;
        for (int t = 0; t < a.ntaps; t++)
          for (int ch = 0; ch < a.chunks; ch++) {
            mbar_wait(empty0 + 8 * st, ph ^ 1);
            mbar_arrive_expect_tx(full0 + 8 * st, a.a_bytes + a.b_bytes);
            tma_load_4d(smemA + st * a.a_stride, &a.tmA, full0 + 8 * st, ch * a.BK, wbase + a.dw[t], hbase + a.dh[t], tc.img);
            tma_load_3d(smemB + st * a.b_stride, &a.tmB, full0 + 8 * st, ch * a.BK, tc.nt * a.n_tile, a.slab[t]);
            ring_next(st, ph, a.stages);
          }
      }
    }
  } else {
    const int t4 = lane & 3;
    int st = 0;
    uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < a.tg.total; tile += gridDim.x) {
      float acc[NT16 * 8];
      switch (a.KK) {
        case 4: tf_mainloop<NT16, 4>(a, acc, smemA, smemB, full0, empty0, st, ph); break;
        case 2: tf_mainloop<NT16, 2>(a, acc, smemA, smemB, full0, empty0, st, ph); break;
        default: tf_mainloop<NT16, 1>(a, acc, smemA, smemB, full0, empty0, st, ph); break;
      }
      const TileCoord tc = tile_coord(a.tg, tile);
      const int n0 = tc.nt * a.n_tile;
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int row = acc_row(warp >> 2, h);
        const int hl = row / a.BW, wl = row - hl * a.BW;
        const int ho = tc.th * a.BH + hl, wo = tc.tw * a.BW + wl;
        if (hl >= a.BH || ho >= a.Ho || wo >= a.Wo) continue;
        float* orow = a.out + (long long)tc.img * a.o_img + (long long)ho * a.o_row + (long long)wo * a.o_pix + a.o_off + n0;
        const float* rrow = EVAL && a.res ? a.res + (((long long)tc.img * a.Ho + ho) * a.Wo + wo) * a.r_pitch + n0 : nullptr;
#pragma unroll
        for (int J = 0; J < NT16 * 2; J++) {
          const int c = 8 * J + 2 * t4;
          if (n0 + c < a.n_out) {  // n_out is a multiple of 4
            float2 o = make_float2(acc[4 * J + 2 * h], acc[4 * J + 2 * h + 1]);
            if (EVAL) {
              const float2 b = *reinterpret_cast<const float2*>(a.bias + n0 + c);
              o.x += b.x; o.y += b.y;
              if (a.act) { o.x = silu_f(o.x); o.y = silu_f(o.y); }
              if (rrow) {  // the Bottleneck shortcut, `x + cv2(cv1(x))` (Block.cs:606)
                const float2 r = *reinterpret_cast<const float2*>(rrow + c);
                o.x = r.x + o.x; o.y = r.y + o.y;
              }
            } else if (a.bias) {
              const float2 b = *reinterpret_cast<const float2*>(a.bias + n0 + c);
              o.x += b.x; o.y += b.y;
            }
            *reinterpret_cast<float2*>(orow + c) = o;
          }
        }
      }
    }
  }
}

// w (Cout, Cin, k, k) checkpoint layout -> wf [tap][Cout][Cin] (forward B operand: rows = output channels, K = Cin)
//                                        -> wb [tap][Cin][Cout] (dgrad B operand: rows = input channels, K = Cout)
__global__ void tf_pack_weights_kernel(const float* __restrict__ w, float* __restrict__ wf, float* __restrict__ wb, int Cout,
                                       int Cin, int taps) {
  const long long n = (long long)Cout * Cin * taps;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int t = (int)(i % taps);
    const long long q = i / taps;
    const int ci = (int)(q % Cin), co = (int)(q / Cin);
    const float v = w[i];
    if (wf) wf[((size_t)t * Cout + co) * Cin + ci] = v;
    if (wb) wb[((size_t)t * Cin + ci) * Cout + co] = v;
  }
}

// Every dense conv weight of a model in ONE launch (the native training step packs once per step, after the optimizer, instead
// of once per conv call: 158 launches of the kernel above in a YOLOv11s step).  wf / wb use the SAME element offsets as the
// checkpoint-layout tensors inside their flat buffer, so a layer's packed operands sit at WF + off and WB + off.
constexpr int TF_PACK_CHUNK = 4096;
__global__ void __launch_bounds__(256) tf_pack_all_kernel(const float* __restrict__ P, float* __restrict__ WF, float* __restrict__ WB,
                                                          const TfPackDesc* __restrict__ d, int nd) {
  int lo = 0, hi = nd - 1;  // last layer whose first chunk <= blockIdx.x
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (d[mid].chunk0 <= (long long)blockIdx.x) lo = mid; else hi = mid - 1;
  }
  const TfPackDesc L = d[lo];
  const long long n = (long long)L.cout * L.cin * L.taps;
  const long long i0 = ((long long)blockIdx.x - L.chunk0) * TF_PACK_CHUNK;
  const float* w = P + L.off;
  float* wf = WF + L.off;
  float* wb = WB + L.off;
  for (long long i = i0 + threadIdx.x; i < min(n, i0 + TF_PACK_CHUNK); i += 256) {
    const int t = (int)(i % L.taps);
    const long long q = i / L.taps;
    const int ci = (int)(q % L.cin), co = (int)(q / L.cin);
    const float v = w[i];
    wf[((size_t)t * L.cout + co) * L.cin + ci] = v;
    wb[((size_t)t * L.cin + ci) * L.cout + co] = v;
  }
}
long long tf_pack_chunks(int cout, int cin, int taps) { return ((long long)cout * cin * taps + TF_PACK_CHUNK - 1) / TF_PACK_CHUNK; }

// Eval-mode BatchNorm folded into every conv of a model in ONE launch (Conv block in `eval()`, Convs.cs:36-56):
//   wf[tap][co][ci] = w[co][ci][tap] * s[co],  bias[co] = beta[co] - rm[co] * s[co],  s = gamma / sqrt(rv + 1e-3)
// computed in double and rounded to fp32 once, as the engine folds on the host (DESIGN.md §3); explicit _rn intrinsics keep
// the compiler from contracting them into FMAs, so the result is the float64 fold rounded to fp32 bit for bit.  invstd[co] =
// 1 / sqrt(rv + 1e-3) serves the convs without a bias epilogue (stem, depthwise), which apply BatchNorm as a separate pass.
// A descriptor without gamma (a plain Conv2d) packs its weights unscaled.  Block b works on chunk b - chunk0 of the
// descriptor that owns it; chunk 0 of each descriptor also writes the per-channel vectors.
__global__ void __launch_bounds__(256) tf_fold_all_kernel(const TfFoldDesc* __restrict__ d, int nd) {
  int lo = 0, hi = nd - 1;  // last descriptor whose first chunk <= blockIdx.x
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (d[mid].chunk0 <= (long long)blockIdx.x) lo = mid; else hi = mid - 1;
  }
  const TfFoldDesc L = d[lo];
  const long long c0 = (long long)blockIdx.x - L.chunk0;
  auto scale = [&](int co) {
    return L.gamma ? __ddiv_rn((double)L.gamma[co], __dsqrt_rn(__dadd_rn((double)L.rv[co], 1e-3))) : 1.0;
  };
  if (c0 == 0 && L.gamma)
    for (int co = threadIdx.x; co < L.cout; co += 256) {
      const double s = scale(co);
      if (L.bias) L.bias[co] = (float)__dsub_rn((double)L.beta[co], __dmul_rn((double)L.rm[co], s));
      if (L.invstd) L.invstd[co] = (float)__ddiv_rn(1.0, __dsqrt_rn(__dadd_rn((double)L.rv[co], 1e-3)));
    }
  if (!L.wf) return;
  const long long n = (long long)L.cout * L.cin * L.taps;
  const long long i0 = c0 * TF_PACK_CHUNK, i1 = min(n, i0 + TF_PACK_CHUNK);
  // the scales of the output channels this chunk touches (at most one per element), once per channel
  __shared__ double sc[TF_PACK_CHUNK];
  const long long per_co = (long long)L.cin * L.taps;
  const int co0 = (int)(i0 / per_co), nco = (int)((i1 - 1) / per_co) - co0 + 1;
  if (L.gamma)
    for (int j = threadIdx.x; j < nco; j += 256) sc[j] = scale(co0 + j);
  __syncthreads();
  for (long long i = i0 + threadIdx.x; i < i1; i += 256) {
    const int t = (int)(i % L.taps);
    const long long q = i / L.taps;
    const int ci = (int)(q % L.cin), co = (int)(q / L.cin);
    L.wf[((size_t)t * L.cout + co) * L.cin + ci] = L.gamma ? (float)__dmul_rn((double)L.w[i], sc[co - co0]) : L.w[i];
  }
}
long long tf_fold_chunks(const TfFoldDesc& d) { return d.wf ? std::max(1ll, tf_pack_chunks(d.cout, d.cin, d.taps)) : 1; }
int tf_fold_all(const TfFoldDesc* dev_descs, int nd, long long total_chunks, cudaStream_t s) {
  if (nd <= 0 || total_chunks <= 0) return YB_OK;
  tf_fold_all_kernel<<<(unsigned)total_chunks, 256, 0, s>>>(dev_descs, nd);
  YB_CUDA_CHECK(cudaGetLastError());
  return YB_OK;
}
int tf_pack_all(const float* P, float* WF, float* WB, const TfPackDesc* dev_descs, int nd, long long total_chunks, cudaStream_t s) {
  if (nd <= 0 || total_chunks <= 0) return YB_OK;
  tf_pack_all_kernel<<<(unsigned)total_chunks, 256, 0, s>>>(P, WF, WB, dev_descs, nd);
  YB_CUDA_CHECK(cudaGetLastError());
  return YB_OK;
}

// One launch of tf_conv_kernel.  in: NHWC (N, Hi, Wi, Kc) fp32; wpk: [taps][Nc][Kc] fp32; out addressing given by strides.
struct TfLaunch {
  const float* in; int N, Hi, Wi, Kc;
  int in_pitch;      // elements between consecutive pixels of `in` (>= Kc: `in` may be a channel slice of a wider NHWC buffer)
  const float* wpk; int Nc, taps_total;
  float* out; long long o_img, o_row, o_pix, o_off;
  const float* bias;
  bool eval;         // eval epilogue: out = [res +] act(acc + bias)
  const float* res; long long r_pitch; int act;
  int Ho, Wo;        // output position grid
  int in_stride;
  int ntaps; int dh[9], dw[9], slab[9];
  bool flat;         // 1x1 stride 1, dense output: flatten the batch into one position dimension
};

// desc: when set, receives one line describing the launch (yb_debug_conv_tf32)
static int tf_conv_launch(const TfLaunch& L, cudaStream_t s, std::string* desc) {
  const EncodeTiledFn encode = tmap_encode_fn();
  if (!encode) { set_error("cuTensorMapEncodeTiled entry point not found"); return YB_ERR_CUDA; }
  TfArgs a;
  memset(&a, 0, sizeof(a));
  a.out = L.out; a.bias = L.bias;
  a.res = L.res; a.r_pitch = L.r_pitch; a.act = L.act;
  a.o_img = L.o_img; a.o_row = L.o_row; a.o_pix = L.o_pix; a.o_off = L.o_off;
  a.n_out = L.Nc;
  a.in_stride = L.in_stride;
  a.ntaps = L.ntaps;
  for (int t = 0; t < L.ntaps; t++) { a.dh[t] = L.dh[t]; a.dw[t] = L.dw[t]; a.slab[t] = L.slab[t]; }
  a.BK = L.Kc >= 32 ? 32 : (L.Kc >= 16 ? 16 : 8);
  a.chunks = (L.Kc + a.BK - 1) / a.BK;
  a.KK = a.BK / 8;
  const uint32_t row_bytes = a.BK * 4;
  a.layout = row_layout(row_bytes);
  a.sbo16 = (8 * row_bytes) >> 4;
  const CUtensorMapSwizzle swz = row_swizzle(row_bytes);
  a.n_tile = std::min(256, (L.Nc + 15) / 16 * 16);
  const int n_tiles = (L.Nc + a.n_tile - 1) / a.n_tile;
  // One N tile as wide as the layer: narrower tiles would give every SM a tile on the 20 x 20 / 40 x 40 levels, at the price
  // of re-reading the activations once per N tile.
  // The flat map is the NHWC map of one image of 1 x (N * H * W) pixels.
  const int npix = L.N * L.Hi * L.Wi;
  const int imgs = L.flat ? 1 : L.N, Hi = L.flat ? 1 : L.Hi, Wi = L.flat ? npix : L.Wi;
  cuuint32_t box[4], estr[4];
  if (L.flat) {
    a.BW = 128; a.BH = 1;
    a.Ho = 1; a.Wo = npix;
    box[0] = a.BK; box[1] = 128; box[2] = 1; box[3] = 1;
    estr[0] = estr[1] = estr[2] = estr[3] = 1;
  } else {
    a.Ho = L.Ho; a.Wo = L.Wo;
    double best = -1;
    for (int bw = 1; bw <= std::min(L.Wo, 128); bw++) {
      const int bh = std::min(L.Ho, 128 / bw);
      if (bw * L.in_stride > 256 || bh * L.in_stride > 256) continue;
      const double tiles = (double)((L.Wo + bw - 1) / bw) * ((L.Ho + bh - 1) / bh);
      const double eff = (double)L.Wo * L.Ho / (tiles * 128.0);
      if (eff > best + 1e-9 || (eff > best - 1e-9 && bw > a.BW)) { best = eff; a.BW = bw; a.BH = bh; }
    }
    box[0] = a.BK; box[1] = a.BW * L.in_stride; box[2] = a.BH * L.in_stride; box[3] = 1;
    estr[0] = 1; estr[1] = L.in_stride; estr[2] = L.in_stride; estr[3] = 1;
  }
  CUresult cr = tmap_nhwc(&a.tmA, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, const_cast<float*>(L.in), 0, L.Kc, Wi, Hi, imgs,
                          L.in_pitch ? L.in_pitch : L.Kc, box, estr, swz);
  if (cr != CUDA_SUCCESS) { set_error("tf32 conv: cuTensorMapEncodeTiled(A) failed with code " + std::to_string((int)cr)); return YB_ERR_CUDA; }
  {
    cuuint64_t bd[3] = {(cuuint64_t)L.Kc, (cuuint64_t)L.Nc, (cuuint64_t)L.taps_total};
    cuuint64_t bs[2] = {(cuuint64_t)L.Kc * 4, (cuuint64_t)L.Kc * 4 * L.Nc};
    cuuint32_t bb[3] = {(cuuint32_t)a.BK, (cuuint32_t)a.n_tile, 1};
    cuuint32_t be[3] = {1, 1, 1};
    cr = encode(&a.tmB, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(L.wpk), bd, bs, bb, be, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) { set_error("tf32 conv: cuTensorMapEncodeTiled(B) failed with code " + std::to_string((int)cr)); return YB_ERR_CUDA; }
  }
  a.tg = tile_grid(imgs, a.Ho, a.Wo, a.BH, a.BW, n_tiles);
  a.a_bytes = (uint32_t)(a.BW * a.BH) * row_bytes;  // the box has BW*BH <= 128 rows; rows past it are never stored
  a.b_bytes = (uint32_t)a.n_tile * row_bytes;
  a.a_stride = (128 * row_bytes + 1023) / 1024 * 1024;
  a.b_stride = (a.n_tile * row_bytes + 1023) / 1024 * 1024;
  // Two CTAs per SM when there are tiles for them and a CTA fits half an SM (n_tile <= 64: 32 accumulator registers per
  // thread, a ring of >= 3 stages in ~100 KiB): the consumers stall in the epilogue of every tile, and a second CTA fills
  // the other's load -> MMA -> epilogue bubbles, as in conv_tc_kernel.
  const size_t per_stage = (size_t)a.a_stride + a.b_stride;
  int occ = 1;
  if (a.n_tile <= 64 && (size_t)(100 * 1024) / per_stage >= 3 && a.tg.total >= 2 * sm_count()) occ = 2;
  a.stages = (int)std::min<size_t>(TF_MAX_STAGES, (size_t)((occ == 2 ? 100 : 190) * 1024) / per_stage);
  if (a.stages < 2) { set_error("tf32 conv: tile does not fit in shared memory"); return YB_ERR_SHAPE; }
  const size_t smem = (size_t)a.stages * (a.a_stride + a.b_stride) + 1024;
  void (*kernel)(TfArgs) = nullptr;
  dispatch_nt16(a.n_tile / 16, [&](auto nt16) {
    kernel = L.eval ? tf_conv_kernel<decltype(nt16)::value, true> : tf_conv_kernel<decltype(nt16)::value, false>;
  });
  YB_CUDA_CHECK(smem_limit((const void*)kernel, smem, false));
  const int grid = std::min(a.tg.total, occ * sm_count());
  if (desc) {
    char line[256];
    snprintf(line, sizeof(line), "%stf_conv_kernel%s BK %d chunks %d n_tile %d x%d BW %d BH %d in_stride %d flat %d ntaps %d occ %d stages %d grid %d",
             desc->empty() ? "" : "\n", L.eval ? "_eval" : "", a.BK, a.chunks, a.n_tile, a.tg.n_tiles, a.BW, a.BH, a.in_stride, L.flat ? 1 : 0,
             a.ntaps, occ, a.stages, grid);
    *desc += line;
  }
  YB_CUDA_CHECK(launch_pdl(kernel, dim3(grid), dim3(TF_THREADS), smem, s, a));
  return 0;
}

static bool tf_shape_ok(int Cin, int Cout, int k, int stride, int pad) {
  return Cin % 8 == 0 && Cout % 8 == 0 && (k == 1 || k == 3) && (stride == 1 || stride == 2) && pad == k / 2;
}

int tf_conv_forward(const float* x, const float* w, const float* bias, int N, int H, int W, int Cin, int Cout, int k, int stride,
                    int pad, float* z, float* ws, size_t ws_bytes, cudaStream_t s, int x_pitch, const float* prepacked,
                    std::string* desc) {
  if (x_pitch && (x_pitch < Cin || x_pitch % 4 || ((uintptr_t)x & 15))) { set_error("tf32 conv: input view must be 16-byte aligned with a pitch multiple of 4"); return YB_ERR_SHAPE; }
  if (!tf_shape_ok(Cin, Cout, k, stride, pad)) { set_error("tf32 conv: channels must be multiples of 8, k in {1,3}, stride in {1,2}, pad = k/2"); return YB_ERR_SHAPE; }
  const size_t wn = (size_t)Cout * Cin * k * k;
  if (!prepacked) {  // prepacked: [tap][Cout][Cin], e.g. from tf_pack_all
    if (ws_bytes < wn * 4) { set_error("tf32 conv forward: workspace too small"); return YB_ERR_INVALID_ARG; }
    tf_pack_weights_kernel<<<(unsigned)std::min<size_t>((wn + 255) / 256, 1024), 256, 0, s>>>(w, ws, nullptr, Cout, Cin, k * k);
  }
  TfLaunch L;
  memset(&L, 0, sizeof(L));
  L.in = x; L.N = N; L.Hi = H; L.Wi = W; L.Kc = Cin; L.in_pitch = x_pitch;
  L.wpk = prepacked ? prepacked : ws; L.Nc = Cout; L.taps_total = k * k;
  L.Ho = (H + 2 * pad - k) / stride + 1; L.Wo = (W + 2 * pad - k) / stride + 1;
  L.out = z; L.o_pix = Cout; L.o_row = (long long)L.Wo * Cout; L.o_img = (long long)L.Ho * L.o_row; L.o_off = 0;
  L.bias = bias;
  L.in_stride = stride;
  L.ntaps = k * k;
  for (int t = 0; t < k * k; t++) { L.dh[t] = t / k - pad; L.dw[t] = t % k - pad; L.slab[t] = t; }
  L.flat = (k == 1 && stride == 1);
  return tf_conv_launch(L, s, desc);
}

int tf_conv_forward_eval(const float* x, int x_pitch, const float* wf, const float* bias, int N, int H, int W, int Cin, int Cout, int k,
                         int stride, int act, const float* res, int res_pitch, float* out, int out_pitch, int out_coff, cudaStream_t s,
                         std::string* desc) {
  auto view_ok = [](const void* p, int pitch, int C) { return pitch >= C && pitch % 4 == 0 && ((uintptr_t)p & 15) == 0; };
  if (!view_ok(x, x_pitch, Cin) || !view_ok(out, out_pitch, out_coff + Cout) || out_coff < 0 || out_coff % 4 || (res && !view_ok(res, res_pitch, Cout))) {
    set_error("tf32 eval conv: input / output / residual views must be 16-byte aligned with pitches and channel offset multiples of 4");
    return YB_ERR_SHAPE;
  }
  if (!tf_shape_ok(Cin, Cout, k, stride, k / 2)) { set_error("tf32 eval conv: channels must be multiples of 8, k in {1,3}, stride in {1,2}"); return YB_ERR_SHAPE; }
  const int pad = k / 2;
  TfLaunch L;
  memset(&L, 0, sizeof(L));
  L.in = x; L.N = N; L.Hi = H; L.Wi = W; L.Kc = Cin; L.in_pitch = x_pitch;
  L.wpk = wf; L.Nc = Cout; L.taps_total = k * k;
  L.Ho = (H + 2 * pad - k) / stride + 1; L.Wo = (W + 2 * pad - k) / stride + 1;
  L.out = out; L.o_pix = out_pitch; L.o_row = (long long)L.Wo * out_pitch; L.o_img = (long long)L.Ho * L.o_row; L.o_off = out_coff;
  L.bias = bias;
  L.eval = true; L.res = res; L.r_pitch = res_pitch; L.act = act;
  L.in_stride = stride;
  L.ntaps = k * k;
  for (int t = 0; t < k * k; t++) { L.dh[t] = t / k - pad; L.dw[t] = t % k - pad; L.slab[t] = t; }
  L.flat = (k == 1 && stride == 1);  // positions are addressed through the pitches, so views flatten like dense tensors
  return tf_conv_launch(L, s, desc);
}

int tf_conv_backward_data(const float* dz, const float* w, int N, int H, int W, int Cin, int Cout, int k, int stride, int pad,
                          float* dx, float* ws, size_t ws_bytes, cudaStream_t s, const float* prepacked,
                          std::string* desc) {
  if (!tf_shape_ok(Cin, Cout, k, stride, pad) || (stride == 2 && ((H | W) & 1))) {
    set_error("tf32 dgrad: channels must be multiples of 8, k in {1,3}, stride in {1,2} (even size for stride 2), pad = k/2");
    return YB_ERR_SHAPE;
  }
  const size_t wn = (size_t)Cout * Cin * k * k;
  if (!prepacked) {  // prepacked: [tap][Cin][Cout]
    if (ws_bytes < wn * 4) { set_error("tf32 dgrad: workspace too small"); return YB_ERR_INVALID_ARG; }
    tf_pack_weights_kernel<<<(unsigned)std::min<size_t>((wn + 255) / 256, 1024), 256, 0, s>>>(w, nullptr, ws, Cout, Cin, k * k);
  }
  const int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
  TfLaunch L;
  memset(&L, 0, sizeof(L));
  L.in = dz; L.N = N; L.Hi = Ho; L.Wi = Wo; L.Kc = Cout;
  L.wpk = prepacked ? prepacked : ws; L.Nc = Cin; L.taps_total = k * k;
  L.out = dx; L.bias = nullptr;
  L.in_stride = 1;
  if (stride == 1) {
    L.Ho = H; L.Wo = W;
    L.o_pix = Cin; L.o_row = (long long)W * Cin; L.o_img = (long long)H * L.o_row; L.o_off = 0;
    L.ntaps = k * k;
    for (int t = 0; t < k * k; t++) { L.dh[t] = pad - t / k; L.dw[t] = pad - t % k; L.slab[t] = t; }
    L.flat = (k == 1);
    return tf_conv_launch(L, s, desc);
  }
  // stride 2: dx(2a + py, 2b + px) = sum over taps with (py + pad - kh), (px + pad - kw) even of dz(a + (py+pad-kh)/2, b + ...)
  // k = 1 (pad 0): only parity (0,0) receives gradient; the other positions are zero.
  if (k == 1) YB_CUDA_CHECK(cudaMemsetAsync(dx, 0, (size_t)N * H * W * Cin * sizeof(float), s));
  for (int py = 0; py < 2; py++)
    for (int px = 0; px < 2; px++) {
      L.ntaps = 0;
      for (int kh = 0; kh < k; kh++)
        for (int kw = 0; kw < k; kw++) {
          const int eh = py + pad - kh, ew = px + pad - kw;
          if ((eh & 1) || (ew & 1)) continue;
          // arithmetic shift: eh in {-1..2} is even here, so eh / 2 is exact for 0 and 2; eh = -2 cannot occur (kh <= 2, pad = 1)
          L.dh[L.ntaps] = eh / 2; L.dw[L.ntaps] = ew / 2; L.slab[L.ntaps] = kh * k + kw;
          L.ntaps++;
        }
      if (L.ntaps == 0) continue;  // k = 1, odd parity: stays zero
      L.Ho = H / 2; L.Wo = W / 2;
      L.o_pix = 2LL * Cin; L.o_row = 2LL * W * Cin; L.o_img = (long long)H * W * Cin;
      L.o_off = ((long long)py * W + px) * Cin;
      L.flat = false;
      const int rc = tf_conv_launch(L, s, desc);
      if (rc) return rc;
    }
  return 0;
}

// ------------------------------------------------------------------------------------------
// weight gradient
// ------------------------------------------------------------------------------------------
constexpr int WG_PW = 8, WG_PH = 8;          // pixel tile of the dz grid (64 pixels = 8 MMAs of K = 8)
constexpr int WG_BLK = WG_PW * WG_PH * 128;  // bytes of one 32-channel block of a pixel tile (64 rows x 128 B)
constexpr int WG_A_STAGES = 2;

struct WgArgs {
  CUtensorMap tmDz, tmX;
  float* part;      // [split][co_pad][tap][ci_pad]
  int Cout, Cin, taps, ksz, stride, pad;
  int nb;           // 32-channel input blocks per CTA (N = nb * 32 columns per tap)
  int co_blocks;    // 32-channel output blocks loaded per CTA (<= 4)
  int co_tiles, ci_tiles, splits;
  int tpc, tap_groups;  // taps per CTA (3 = one kh row of a 3x3, 1 for 1x1) and groups of them
  TileGrid tg;       // pixel tiles of the dz grid (n_tiles = 1)
  int b_stages;
  int halo;         // 3x3 stride 1: ONE PH x (PW+2) input tile per pixel tile serves the three taps of a kh row (row-shifted windows)
  uint32_t xblk;    // bytes reserved per 32-channel block of an x stage (1 KiB aligned)
  int co_pad, ci_pad;
};

// fp32 element (row r, channel c < 32) of a 128-byte-row SWIZZLE_128B tile whose base is 1 KiB aligned
__device__ __forceinline__ uint32_t wg_ld(uint32_t base, int r, int c) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(base + r * 128 + ((((c >> 2) ^ (r & 7)) << 4) | ((c & 3) << 2))));
  return v;
}
__device__ __forceinline__ void mma_tf32_16x8x8(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__global__ void __launch_bounds__(TF_THREADS, 1) tf_wgrad_kernel(const __grid_constant__ WgArgs a) {
  extern __shared__ __align__(1024) uint8_t wg_smem[];
  __shared__ __align__(8) uint64_t bars[2 * WG_A_STAGES + 2 * 16];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t smem0 = (smem_u32(wg_smem) + 1023u) & ~1023u;
  const uint32_t a_stride = 4 * WG_BLK, b_stride = (uint32_t)a.nb * a.xblk;
  const uint32_t smemA = smem0, smemB = smem0 + WG_A_STAGES * a_stride;
  const uint32_t afull = smem_u32(&bars[0]), aempty = smem_u32(&bars[WG_A_STAGES]);
  const uint32_t bfull = smem_u32(&bars[2 * WG_A_STAGES]), bempty = smem_u32(&bars[2 * WG_A_STAGES + 16]);
  if (threadIdx.x == 0) {
    for (int s = 0; s < WG_A_STAGES; s++) { mbar_init(afull + 8 * s, 1); mbar_init(aempty + 8 * s, TF_CONSUMER_WARPS); }
    for (int s = 0; s < a.b_stages; s++) { mbar_init(bfull + 8 * s, 1); mbar_init(bempty + 8 * s, TF_CONSUMER_WARPS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  // rows of the dz stages that are never loaded (Cout < 128) feed accumulator rows that are never stored; zero them anyway
  // so that no NaN / denormal bit patterns reach the tensor cores
  for (uint32_t i = threadIdx.x; i < WG_A_STAGES * a_stride / 16; i += TF_THREADS) st_shared_v4(smemA + i * 16, make_int4(0, 0, 0, 0));
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  pdl_wait();
  pdl_trigger();

  // CTA -> (output-channel tile, input-channel tile, pixel split)
  const int split = blockIdx.x % a.splits;
  const int rest = blockIdx.x / a.splits;
  const int tg = rest % a.tap_groups, pair = rest / a.tap_groups;
  const int ci_t = pair % a.ci_tiles, co_t = pair / a.ci_tiles;
  const int tap0 = tg * a.tpc;
  const int my_tiles = split < a.tg.total ? (a.tg.total - split + a.splits - 1) / a.splits : 0;
  const int ncols = a.nb * 32;  // accumulator columns per tap

  if (warp == TF_CONSUMER_WARPS) {
    if (lane == 0) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&a.tmDz) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&a.tmX) : "memory");
      int sa = 0, sb = 0;
      uint32_t pa = 0, pb = 0;
      for (int i = 0; i < my_tiles; i++) {
        const TileCoord tc = tile_coord(a.tg, split + i * a.splits);
        const int w0 = tc.tw * WG_PW, h0 = tc.th * WG_PH;
        mbar_wait(aempty + 8 * sa, pa ^ 1);
        mbar_arrive_expect_tx(afull + 8 * sa, (uint32_t)a.co_blocks * WG_BLK);
        for (int b = 0; b < a.co_blocks; b++)
          tma_load_4d(smemA + sa * a_stride + b * WG_BLK, &a.tmDz, afull + 8 * sa, co_t * 128 + b * 32, w0, h0, tc.img);
        ring_next(sa, pa, WG_A_STAGES);
        if (a.halo) {
          // one box of PH x (PW + 2) input pixels per 32-channel block for the kh row of this CTA: tap (kh, kw) of output
          // row h reads its 8 pixels from rows h * (PW + 2) + kw .. + 7 of it
          const int kh = tap0 / 3;
          mbar_wait(bempty + 8 * sb, pb ^ 1);
          mbar_arrive_expect_tx(bfull + 8 * sb, (uint32_t)a.nb * (WG_PW + 2) * WG_PH * 128);
          for (int b = 0; b < a.nb; b++)
            tma_load_4d(smemB + sb * b_stride + b * a.xblk, &a.tmX, bfull + 8 * sb, (ci_t * a.nb + b) * 32, w0 - a.pad, h0 + kh - a.pad, tc.img);
          ring_next(sb, pb, a.b_stages);
        } else {
          for (int tt = 0; tt < a.tpc; tt++) {
            const int t = tap0 + tt;
            const int kh = t / a.ksz, kw = t - kh * a.ksz;
            mbar_wait(bempty + 8 * sb, pb ^ 1);
            mbar_arrive_expect_tx(bfull + 8 * sb, (uint32_t)a.nb * WG_BLK);
            for (int b = 0; b < a.nb; b++)
              tma_load_4d(smemB + sb * b_stride + b * a.xblk, &a.tmX, bfull + 8 * sb, (ci_t * a.nb + b) * 32,
                          w0 * a.stride + kw - a.pad, h0 * a.stride + kh - a.pad, tc.img);
            ring_next(sb, pb, a.b_stages);
          }
        }
      }
    }
  } else {
    // warp w: output channels 16w .. 16w+15 of the CTA's 128 (A rows) and every accumulator column; column block j (8
    // columns) is tap j / (nb * 4), input channels 8 * (j % (nb * 4)) ..  At most 128 columns: 16 blocks x 4 registers.
    const int g = lane >> 2, t4 = lane & 3;
    const int nblk = a.tpc * a.nb * 4;
    const int acol = 16 * (warp & 1) + g;  // channel of this lane's A rows inside 32-channel block warp / 2
    float acc[16][4];
#pragma unroll
    for (int j = 0; j < 16; j++) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
    int sa = 0, sb = 0;
    uint32_t pa = 0, pb = 0;
    const int nst = a.halo ? 1 : a.tpc;  // B stages per pixel tile
    for (int i = 0; i < my_tiles; i++) {
      mbar_wait(afull + 8 * sa, pa);
      const uint32_t A0 = smemA + sa * a_stride + (warp >> 1) * WG_BLK;
      uint32_t B0[3];
#pragma unroll
      for (int q = 0; q < 3; q++) {
        const int sq = sb + q < a.b_stages ? sb + q : sb + q - a.b_stages;
        if (q < nst) mbar_wait(bfull + 8 * sq, sb + q < a.b_stages ? pb : (pb ^ 1));
        B0[q] = smemB + (q < nst ? sq : sb) * b_stride;
      }
      for (int ks = 0; ks < WG_PW * WG_PH / 8; ks++) {  // 8 pixels = one pixel row of the tile per K step
        uint32_t af[4];
        af[0] = wg_ld(A0, 8 * ks + t4, acol);
        af[1] = wg_ld(A0, 8 * ks + t4, acol + 8);
        af[2] = wg_ld(A0, 8 * ks + t4 + 4, acol);
        af[3] = wg_ld(A0, 8 * ks + t4 + 4, acol + 8);
#pragma unroll
        for (int j = 0; j < 16; j++) {
          if (j < nblk) {
            const int tt = a.tpc == 3 ? (j >> 2) : 0, jj = a.tpc == 3 ? (j & 3) : j;  // tpc = 3 implies nb = 1
            const uint32_t bb = (a.halo ? B0[0] : B0[tt]) + (jj >> 2) * a.xblk;
            // halo: output row ks reads input pixels ks * (PW + 2) + kw .. of the box
            const int r0 = a.halo ? ks * (WG_PW + 2) + t4 + tt : 8 * ks + t4;
            const int c = (jj & 3) * 8 + g;
            mma_tf32_16x8x8(acc[j], af, wg_ld(bb, r0, c), wg_ld(bb, r0 + 4, c));
          }
        }
      }
      __syncwarp();  // every lane's shared-memory reads of this tile are done
      if (lane == 0) {
        mbar_arrive(aempty + 8 * sa);
        for (int q = 0; q < nst; q++) mbar_arrive(bempty + 8 * (sb + q < a.b_stages ? sb + q : sb + q - a.b_stages));
      }
      ring_next(sa, pa, WG_A_STAGES);
      for (int q = 0; q < nst; q++) ring_next(sb, pb, a.b_stages);
    }
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int co = co_t * 128 + warp * 16 + g + 8 * h;
      if (co >= a.Cout) continue;
      float* prow = a.part + (((size_t)split * a.co_pad + co) * a.taps) * a.ci_pad + (size_t)ci_t * ncols;
#pragma unroll
      for (int j = 0; j < 16; j++) {
        if (j < nblk) {
          const int tt = a.tpc == 3 ? (j >> 2) : 0, jj = a.tpc == 3 ? (j & 3) : j;
          *reinterpret_cast<float2*>(prow + (size_t)(tap0 + tt) * a.ci_pad + 8 * jj + 2 * t4) = make_float2(acc[j][2 * h], acc[j][2 * h + 1]);
        }
      }
    }
  }
}

// dw[co][ci][tap] = sum over splits (fixed order) of part[split][co][tap][ci]
// One block per output channel: the partials are read along ci (coalesced), summed over the splits in split order, transposed
// through shared memory ([ci][tap], stride `taps` is odd or 1: no bank conflicts) and written as the contiguous run
// dw[co][:][:].  (Threads over the checkpoint layout would read 4-byte words ci_pad apart.)
__global__ void __launch_bounds__(256) tf_wgrad_fold_kernel(const float* __restrict__ part, float* __restrict__ dw, int Cout, int Cin,
                                                            int taps, int splits, int co_pad, int ci_pad) {
  pdl_wait();
  pdl_trigger();
  extern __shared__ float fold_sm[];  // [Cin][taps]
  const int co = blockIdx.x;
  const size_t ss = (size_t)co_pad * taps * ci_pad;
  const float* base = part + (size_t)co * taps * ci_pad;
  const int n = Cin * taps;
  for (int e = threadIdx.x; e < n; e += 256) {
    const int t = e / Cin, ci = e - t * Cin;
    const float* p = base + (size_t)t * ci_pad + ci;
    float acc = 0.f;
    int sp = 0;
    for (; sp + 4 <= splits; sp += 4) {
      const float a0 = p[(size_t)sp * ss], a1 = p[(size_t)(sp + 1) * ss], a2 = p[(size_t)(sp + 2) * ss], a3 = p[(size_t)(sp + 3) * ss];
      acc += a0; acc += a1; acc += a2; acc += a3;
    }
    for (; sp < splits; sp++) acc += p[(size_t)sp * ss];
    fold_sm[ci * taps + t] = acc;
  }
  __syncthreads();
  float* out = dw + (size_t)co * n;
  for (int e = threadIdx.x; e < n; e += 256) out[e] = fold_sm[e];
}

struct WgPlan { int nb, co_tiles, ci_tiles, splits, co_pad, ci_pad, tpc, tap_groups; TileGrid tg; };
static WgPlan wg_plan(int N, int H, int W, int Cin, int Cout, int k, int stride, int pad) {
  WgPlan p;
  const int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
  const int taps = k * k;
  const int ci_blocks = (Cin + 31) / 32;
  // a CTA owns 128 output channels x (tpc taps x nb * 32 input channels) of accumulators in registers, at most 128
  // columns: tpc = 3 (one kh row of a 3x3) x 32 channels, or one tap x up to 128 channels
  p.tpc = taps == 9 ? 3 : 1;
  p.nb = std::min(ci_blocks, p.tpc == 3 ? 1 : 4);
  p.ci_tiles = (ci_blocks + p.nb - 1) / p.nb;
  p.co_tiles = (Cout + 127) / 128;
  p.co_pad = p.co_tiles * 128;
  p.ci_pad = p.ci_tiles * p.nb * 32;
  p.tg = tile_grid(N, Ho, Wo, WG_PH, WG_PW, 1);
  p.tap_groups = taps / p.tpc;
  const int pairs = p.co_tiles * p.ci_tiles * p.tap_groups;
  // pixel splits: one CTA per SM (189 KiB of shared memory), so the grid should fill ONE wave of SMs, or two when that fills
  // them noticeably better - never a few CTAs over (ceil(2 * SMs / pairs) capped at 64 gave grids of 300 - 320 = a third
  // wave of 4 - 24 CTAs on a third of the layers, and 64-CTA grids on the 1x1 layers with <= 128 channels)
  const int sms = sm_count();
  const int s1 = std::max(1, sms / pairs), s2 = std::max(1, 2 * sms / pairs);
  const double u1 = (double)std::min(pairs * s1, sms) / sms, u2 = (double)std::min(pairs * s2, 2 * sms) / (2.0 * sms);
  p.splits = (pairs <= sms && u2 > u1 + 0.08) ? s2 : s1;
  p.splits = std::max(1, std::min(p.splits, p.tg.total));
  return p;
}

size_t tf_conv_workspace_bytes(int N, int H, int W, int Cin, int Cout, int k, int stride) {
  const WgPlan p = wg_plan(N, H, W, Cin, Cout, k, stride, k / 2);
  const size_t part = (size_t)p.splits * p.co_pad * k * k * p.ci_pad * 4;
  const size_t wpk = (size_t)Cout * Cin * k * k * 4;
  return std::max(std::max(part, wpk), (size_t)ST_WG_BLOCKS * 27 * 128 * sizeof(float)) + 256;
}

int tf_conv_backward_weight(const float* x, const float* dz, int N, int H, int W, int Cin, int Cout, int k, int stride, int pad,
                            float* dw, float* ws, size_t ws_bytes, cudaStream_t s, int x_pitch, std::string* desc) {
  if (x_pitch && (x_pitch < Cin || x_pitch % 4 || ((uintptr_t)x & 15))) { set_error("tf32 wgrad: input view must be 16-byte aligned with a pitch multiple of 4"); return YB_ERR_SHAPE; }
  const int xp = x_pitch ? x_pitch : Cin;
  if (!tf_shape_ok(Cin, Cout, k, stride, pad)) { set_error("tf32 wgrad: channels must be multiples of 8, k in {1,3}, stride in {1,2}, pad = k/2"); return YB_ERR_SHAPE; }
  if (!tmap_encode_fn()) { set_error("cuTensorMapEncodeTiled entry point not found"); return YB_ERR_CUDA; }
  const WgPlan p = wg_plan(N, H, W, Cin, Cout, k, stride, pad);
  const size_t part_bytes = (size_t)p.splits * p.co_pad * k * k * p.ci_pad * 4;
  if (ws_bytes < part_bytes) { set_error("tf32 wgrad: workspace too small"); return YB_ERR_INVALID_ARG; }
  const int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
  WgArgs a;
  memset(&a, 0, sizeof(a));
  a.part = ws;
  a.Cout = Cout; a.Cin = Cin; a.taps = k * k; a.ksz = k; a.stride = stride; a.pad = pad;
  a.nb = p.nb; a.co_tiles = p.co_tiles; a.ci_tiles = p.ci_tiles; a.splits = p.splits;
  a.tpc = p.tpc; a.tap_groups = p.tap_groups;
  a.co_blocks = std::min(4, (Cout + 31) / 32);
  a.tg = p.tg;
  a.co_pad = p.co_pad; a.ci_pad = p.ci_pad;
  // 3x3 stride 1: the input tile with its halo is loaded once per pixel tile and the nine taps are row-shifted MMA windows
  // into it (the per-tap form moved 9 x 8 KiB of x per 64 pixels and was bound by L2 -> SM delivery).
  a.halo = (k == 3 && stride == 1) ? 1 : 0;
  a.xblk = a.halo ? (uint32_t)(((WG_PW + 2) * WG_PH * 128 + 1023) / 1024 * 1024) : (uint32_t)WG_BLK;
  const size_t b_stride = (size_t)p.nb * a.xblk;
  a.b_stages = (int)std::min<size_t>(16, ((size_t)190 * 1024 - (size_t)WG_A_STAGES * 4 * WG_BLK) / b_stride);
  if (a.b_stages < 2) { set_error("tf32 wgrad: tile does not fit in shared memory"); return YB_ERR_SHAPE; }
  {
    const cuuint32_t bx[4] = {32, WG_PW, WG_PH, 1}, es[4] = {1, 1, 1, 1};
    const CUresult cr = tmap_nhwc(&a.tmDz, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, const_cast<float*>(dz), 0, Cout, Wo, Ho, N, Cout, bx, es,
                                  CU_TENSOR_MAP_SWIZZLE_128B);
    if (cr != CUDA_SUCCESS) { set_error("tf32 wgrad: cuTensorMapEncodeTiled(dz) failed with code " + std::to_string((int)cr)); return YB_ERR_CUDA; }
  }
  {
    const cuuint32_t bx[4] = {32, (cuuint32_t)(a.halo ? WG_PW + 2 : WG_PW * stride), (cuuint32_t)(a.halo ? WG_PH : WG_PH * stride), 1};
    const cuuint32_t es[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
    const CUresult cr = tmap_nhwc(&a.tmX, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, const_cast<float*>(x), 0, Cin, W, H, N, xp, bx, es,
                                  CU_TENSOR_MAP_SWIZZLE_128B);
    if (cr != CUDA_SUCCESS) { set_error("tf32 wgrad: cuTensorMapEncodeTiled(x) failed with code " + std::to_string((int)cr)); return YB_ERR_CUDA; }
  }
  const size_t smem = (size_t)WG_A_STAGES * 4 * WG_BLK + (size_t)a.b_stages * b_stride + 1024;
  YB_CUDA_CHECK(smem_limit((const void*)tf_wgrad_kernel, smem, false));
  const int grid = p.co_tiles * p.ci_tiles * p.tap_groups * p.splits;
  if (desc) {
    char line[256];
    snprintf(line, sizeof(line), "%stf_wgrad_kernel halo %d tpc %d nb %d co_tiles %d ci_tiles %d co_blocks %d splits %d pix_tiles %d b_stages %d grid %d",
             desc->empty() ? "" : "\n", a.halo, a.tpc, a.nb, a.co_tiles, a.ci_tiles, a.co_blocks, a.splits, a.tg.total, a.b_stages, grid);
    *desc += line;
  }
  YB_CUDA_CHECK(launch_pdl(tf_wgrad_kernel, dim3(grid), dim3(TF_THREADS), smem, s, a));
  const size_t fold_smem = (size_t)Cin * k * k * sizeof(float);
  if (fold_smem > (size_t)160 * 1024) { set_error("tf32 wgrad: Cin * k * k too large for the fold"); return YB_ERR_SHAPE; }
  YB_CUDA_CHECK(smem_limit((const void*)tf_wgrad_fold_kernel, fold_smem, false));
  YB_CUDA_CHECK(launch_pdl(tf_wgrad_fold_kernel, dim3(Cout), dim3(256), fold_smem, s, (const float*)ws, dw, Cout, Cin, k * k,
                           p.splits, p.co_pad, p.ci_pad));
  YB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------
// The 3-channel stem (model.0: Conv(3, C, k = 3, s = 2), Yolo.cs:53) on CUDA cores, fp32.
// On the tensor cores the stem would need its input zero-padded to 8 channels: K = 8 per tap means one tiny MMA per TMA
// box of 128 strided 32-byte rows, bound by the TMA row rate, for 0.3 % of the step's FLOPs.  Here:
//   forward   one thread per output pixel and 32-channel group: its 27 inputs in registers, weights [27][C] in shared memory
//   wgrad     dW[co][ci][kh][kw] = sum over pixels of dz[p][co] * x[window(p)][ci][kh][kw]: a block stages 128 pixels (their
//             27-value windows and dz rows) in shared memory, thread (co lane, tap group) accumulates its share of the
//             27 x C products; per-block partials are folded in block order (deterministic)
// x is NHWC with `xc` channels per pixel of which the first 3 are used (the native step keeps an 8-channel input).
// ------------------------------------------------------------------------------------------
constexpr int ST_PIX = 128;

__global__ void __launch_bounds__(256) stem3_forward_kernel(const float* __restrict__ x, int xc, const float* __restrict__ w,
                                                           float* __restrict__ z, int N, int H, int W, int Ho, int Wo, int C) {
  extern __shared__ float sw[];  // [27][C]: k = (kh * 3 + kw) * 3 + ci
  for (int i = threadIdx.x; i < 27 * C; i += blockDim.x) {
    const int co = i % C, k = i / C;
    const int ci = k % 3, t = k / 3;
    sw[i] = w[(co * 3 + ci) * 9 + t];
  }
  __syncthreads();
  const int groups = (C + 31) / 32;
  const long long total = (long long)N * Ho * Wo * groups;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(idx % groups);
    long long p = idx / groups;
    const int wo = (int)(p % Wo);
    p /= Wo;
    const int ho = (int)(p % Ho);
    const int n = (int)(p / Ho);
    float in[27];
#pragma unroll
    for (int kh = 0; kh < 3; kh++) {
      const int hi = 2 * ho + kh - 1;
#pragma unroll
      for (int kw = 0; kw < 3; kw++) {
        const int wi = 2 * wo + kw - 1;
        const bool ok = hi >= 0 && hi < H && wi >= 0 && wi < W;
        const float* px = x + (((size_t)n * H + (ok ? hi : 0)) * W + (ok ? wi : 0)) * xc;
#pragma unroll
        for (int ci = 0; ci < 3; ci++) in[(kh * 3 + kw) * 3 + ci] = ok ? px[ci] : 0.f;
      }
    }
    const int c0 = g * 32, cn = min(32, C - c0);
    float* out = z + ((size_t)(n * Ho + ho) * Wo + wo) * C + c0;
    for (int c = 0; c < cn; c += 4) {  // C is a multiple of 8
      float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
      for (int k = 0; k < 27; k++) {
        const float4 wv = *reinterpret_cast<const float4*>(sw + k * C + c0 + c);
        a0 = fmaf(in[k], wv.x, a0); a1 = fmaf(in[k], wv.y, a1); a2 = fmaf(in[k], wv.z, a2); a3 = fmaf(in[k], wv.w, a3);
      }
      *reinterpret_cast<float4*>(out + c) = make_float4(a0, a1, a2, a3);
    }
  }
}

// Row-segment version: a tile is up to 128 adjacent output pixels of one output row.  The three input rows it needs are staged
// as [kh][column][4] (one 16-byte load per input pixel, coalesced), so the 3 x 3 window of output pixel p is 3 x three
// adjacent float4 of shared memory; dz of the tile is staged as [pixel][C].  Thread = (channel lane, warp g): warp g takes
// pixels g, g + 8, ... and keeps all 27 taps of its channel(s) in registers: per pixel 9 broadcast LDS.128 + 1 LDS feed
// 27 FMAs (staging im2col windows element by element costs ~40 integer instructions per staged value and 5 LDS per
// 4 FMAs).  The 8 warps are folded in warp order through shared memory, the blocks'
// partials by stem3_wgrad_fold_kernel in block order: deterministic.
// grid.x blocks walk the tiles with stride gridDim.x; partial[block][27][C], k = (kh * 3 + kw) * 3 + ci
template <int CG>  // 32-channel groups per thread: ceil(C / 32)
__global__ void __launch_bounds__(256) stem3_wgrad_partial_kernel(const float* __restrict__ x, int xc, const float* __restrict__ dz,
                                                                 float* __restrict__ partial, int N, int H, int W, int Ho, int Wo, int C) {
  extern __shared__ __align__(16) float sm[];
  float* xs = sm;                              // [3][2 * ST_PIX + 1][4]
  float* ds = sm + 3 * (2 * ST_PIX + 1) * 4;   // [ST_PIX][C]; later the fold buffer [8][27][32]
  const int lane = threadIdx.x & 31, g = threadIdx.x >> 5;
  const int segs = (Wo + ST_PIX - 1) / ST_PIX;
  const long long tiles = (long long)N * Ho * segs;
  float acc[CG][27];
#pragma unroll
  for (int b2 = 0; b2 < CG; b2++)
#pragma unroll
    for (int k = 0; k < 27; k++) acc[b2][k] = 0.f;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int seg = (int)(tile % segs);
    const long long q = tile / segs;
    const int ho = (int)(q % Ho), n = (int)(q / Ho);
    const int wo0 = seg * ST_PIX, npx = min(ST_PIX, Wo - wo0);
    const int ncol = 2 * npx + 1, wi0 = 2 * wo0 - 1;
    __syncthreads();
    for (int i = threadIdx.x; i < 3 * ncol; i += 256) {
      const int kh = i / ncol, j = i - kh * ncol;
      const int hi = 2 * ho + kh - 1, wi = wi0 + j;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (hi >= 0 && hi < H && wi >= 0 && wi < W) {
        const float* px = x + (((size_t)n * H + hi) * W + wi) * xc;
        if ((xc & 3) == 0) v = __ldg(reinterpret_cast<const float4*>(px));
        else { v.x = px[0]; v.y = px[1]; v.z = px[2]; }
      }
      *reinterpret_cast<float4*>(xs + ((size_t)kh * (2 * ST_PIX + 1) + j) * 4) = v;
    }
    const float* dzt = dz + (((size_t)n * Ho + ho) * Wo + wo0) * C;  // npx * C contiguous floats (C % 8 == 0: 16-byte aligned)
    for (int i = threadIdx.x; i < npx * C / 4; i += 256)
      *reinterpret_cast<float4*>(ds + (size_t)i * 4) = __ldg(reinterpret_cast<const float4*>(dzt) + i);
    __syncthreads();
    for (int pl = g; pl < npx; pl += 8) {
      float4 w9[9];  // [kh][kw] -> (ci 0..2, pad)
#pragma unroll
      for (int kh = 0; kh < 3; kh++)
#pragma unroll
        for (int kw = 0; kw < 3; kw++)
          w9[kh * 3 + kw] = *reinterpret_cast<const float4*>(xs + ((size_t)kh * (2 * ST_PIX + 1) + 2 * pl + kw) * 4);
#pragma unroll
      for (int b2 = 0; b2 < CG; b2++) {
        {
          const int c = b2 * 32 + lane;
          const float gv = c < C ? ds[pl * C + c] : 0.f;
#pragma unroll
          for (int t = 0; t < 9; t++) {
            acc[b2][t * 3 + 0] = fmaf(gv, w9[t].x, acc[b2][t * 3 + 0]);
            acc[b2][t * 3 + 1] = fmaf(gv, w9[t].y, acc[b2][t * 3 + 1]);
            acc[b2][t * 3 + 2] = fmaf(gv, w9[t].z, acc[b2][t * 3 + 2]);
          }
        }
      }
    }
  }
  // fold the 8 warps in warp order, one 32-channel group at a time
  float* red = ds;  // [8][27][32]
#pragma unroll
  for (int b2 = 0; b2 < CG; b2++) {
    {
      __syncthreads();
#pragma unroll
      for (int k = 0; k < 27; k++) red[(g * 27 + k) * 32 + lane] = acc[b2][k];
      __syncthreads();
      for (int i = threadIdx.x; i < 27 * 32; i += 256) {
        const int k = i >> 5, cl = i & 31;
        float sum = 0.f;
        for (int w8 = 0; w8 < 8; w8++) sum += red[(w8 * 27 + k) * 32 + cl];
        const int c = b2 * 32 + cl;
        if (c < C) partial[((size_t)blockIdx.x * 27 + k) * C + c] = sum;
      }
    }
  }
}
__global__ void stem3_wgrad_fold_kernel(const float* __restrict__ partial, int blocks, int C, float* __restrict__ dw) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // (k, c)
  if (i >= 27 * C) return;
  const int k = i / C, c = i - k * C;
  float s = 0.f;
  for (int b = 0; b < blocks; b++) s += partial[((size_t)b * 27 + k) * C + c];
  const int ci = k % 3, t = k / 3;
  dw[(c * 3 + ci) * 9 + t] = s;
}

int stem3_forward(const float* x, int xc, const float* w, int N, int H, int W, int C, float* z, cudaStream_t s) {
  if (C % 8 || C > 128 || (H & 1) || (W & 1) || xc < 3) { set_error("stem conv: C % 8 == 0, C <= 128, even input size"); return YB_ERR_SHAPE; }
  const int Ho = H / 2, Wo = W / 2;
  const long long total = (long long)N * Ho * Wo * ((C + 31) / 32);
  const int grid = (int)std::min<long long>((total + 255) / 256, sm_count() * 16);
  stem3_forward_kernel<<<grid, 256, (size_t)27 * C * sizeof(float), s>>>(x, xc, w, z, N, H, W, Ho, Wo, C);
  YB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
size_t stem3_wgrad_workspace_bytes(int C) { return (size_t)ST_WG_BLOCKS * 27 * C * sizeof(float); }
int stem3_backward_weight(const float* x, int xc, const float* dz, int N, int H, int W, int C, float* dw, float* ws, size_t ws_bytes,
                          cudaStream_t s) {
  if (C % 8 || C > 128 || (H & 1) || (W & 1) || xc < 3) { set_error("stem wgrad: C % 8 == 0, C <= 128, even input size"); return YB_ERR_SHAPE; }
  const int blocks = ST_WG_BLOCKS;
  if (ws_bytes < stem3_wgrad_workspace_bytes(C)) { set_error("stem wgrad: workspace too small"); return YB_ERR_INVALID_ARG; }
  const int Ho = H / 2, Wo = W / 2;
  const size_t smem = (size_t)(3 * (2 * ST_PIX + 1) * 4 + std::max(ST_PIX * C, 8 * 27 * 32)) * sizeof(float);
  const int cg = (C + 31) / 32;
  const auto kernel = cg == 1 ? stem3_wgrad_partial_kernel<1> : cg == 2 ? stem3_wgrad_partial_kernel<2>
                    : cg == 3 ? stem3_wgrad_partial_kernel<3> : stem3_wgrad_partial_kernel<4>;
  YB_CUDA_CHECK(smem_limit((const void*)kernel, smem, false));
  kernel<<<blocks, 256, smem, s>>>(x, xc, dz, ws, N, H, W, Ho, Wo, C);
  stem3_wgrad_fold_kernel<<<(27 * C + 127) / 128, 128, 0, s>>>(ws, blocks, C, dw);
  YB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace yb

using namespace yb;

extern "C" {

int64_t yb_conv_tc_workspace_bytes(int32_t n, int32_t height, int32_t width, int32_t cin, int32_t cout, int32_t k, int32_t stride) {
  if (n <= 0 || height <= 0 || width <= 0 || cin <= 0 || cout <= 0 || k <= 0 || stride <= 0) return 0;
  if (!have_device("yb_conv_tc_workspace_bytes")) return 0;
  return (int64_t)tf_conv_workspace_bytes(n, height, width, cin, cout, k, stride);
}

int32_t yb_conv_forward_tc(const float* x, const float* w, const float* bias, int32_t n, int32_t height, int32_t width, int32_t cin,
                           int32_t cout, int32_t k, int32_t stride, int32_t pad, float* z, void* workspace, int64_t workspace_bytes,
                           void* stream) {
  if (!x || !w || !z || !workspace) { set_error("yb_conv_forward_tc: null argument"); return YB_ERR_INVALID_ARG; }
  if (n <= 0 || height <= 0 || width <= 0 || cin <= 0 || cout <= 0) { set_error("yb_conv_forward_tc: bad shape"); return YB_ERR_SHAPE; }
  if (!have_device("yb_conv_forward_tc")) return YB_ERR_NO_DEVICE;
  return tf_conv_forward(x, w, bias, n, height, width, cin, cout, k, stride, pad, z, (float*)workspace, (size_t)workspace_bytes,
                         (cudaStream_t)stream, 0, nullptr);
}

int32_t yb_conv_backward_data_tc(const float* dz, const float* w, int32_t n, int32_t height, int32_t width, int32_t cin, int32_t cout,
                                 int32_t k, int32_t stride, int32_t pad, float* dx, void* workspace, int64_t workspace_bytes,
                                 void* stream) {
  if (!dz || !w || !dx || !workspace) { set_error("yb_conv_backward_data_tc: null argument"); return YB_ERR_INVALID_ARG; }
  if (n <= 0 || height <= 0 || width <= 0 || cin <= 0 || cout <= 0) { set_error("yb_conv_backward_data_tc: bad shape"); return YB_ERR_SHAPE; }
  if (!have_device("yb_conv_backward_data_tc")) return YB_ERR_NO_DEVICE;
  return tf_conv_backward_data(dz, w, n, height, width, cin, cout, k, stride, pad, dx, (float*)workspace, (size_t)workspace_bytes,
                               (cudaStream_t)stream, nullptr);
}

int32_t yb_conv_backward_weight_tc(const float* x, const float* dz, int32_t n, int32_t height, int32_t width, int32_t cin,
                                   int32_t cout, int32_t k, int32_t stride, int32_t pad, float* dw, void* workspace,
                                   int64_t workspace_bytes, void* stream) {
  if (!x || !dz || !dw || !workspace) { set_error("yb_conv_backward_weight_tc: null argument"); return YB_ERR_INVALID_ARG; }
  if (n <= 0 || height <= 0 || width <= 0 || cin <= 0 || cout <= 0) { set_error("yb_conv_backward_weight_tc: bad shape"); return YB_ERR_SHAPE; }
  if (!have_device("yb_conv_backward_weight_tc")) return YB_ERR_NO_DEVICE;
  return tf_conv_backward_weight(x, dz, n, height, width, cin, cout, k, stride, pad, dw, (float*)workspace, (size_t)workspace_bytes,
                                 (cudaStream_t)stream, 0);
}

int32_t yb_debug_conv_tf32(int32_t pass, const float* x, int32_t x_pitch, const float* dz, const float* w, const float* bias,
                           int32_t n, int32_t height, int32_t width, int32_t cin, int32_t cout, int32_t k, int32_t stride,
                           float* out, void* workspace, int64_t workspace_bytes, char* desc, int32_t desc_capacity) {
  if (pass < 0 || pass > 2) { set_error("yb_debug_conv_tf32: pass must be 0 (forward), 1 (data gradient) or 2 (weight gradient)"); return YB_ERR_INVALID_ARG; }
  if ((pass != 1 && !x) || (pass != 0 && !dz) || (pass != 2 && !w) || !out || !workspace) {
    set_error("yb_debug_conv_tf32: null argument");
    return YB_ERR_INVALID_ARG;
  }
  if (n <= 0 || height <= 0 || width <= 0 || cin <= 0 || cout <= 0 || workspace_bytes <= 0 || x_pitch < 0 ||
      (x_pitch && (pass == 1 || x_pitch < cin || x_pitch % 4 || ((uintptr_t)x & 15)))) {
    set_error("yb_debug_conv_tf32: bad argument (extent, workspace size, or x_pitch: >= cin, a multiple of 4 on a 16-byte aligned "
              "x, and 0 for the data gradient)");
    return YB_ERR_INVALID_ARG;
  }
  if (!tf_shape_ok(cin, cout, k, stride, k / 2) || (pass == 1 && stride == 2 && ((height | width) & 1))) {
    set_error("yb_debug_conv_tf32: shape not supported: channels must be multiples of 8, k in {1,3}, stride in {1,2}, "
              "even extents for a stride-2 data gradient");
    return YB_ERR_SHAPE;
  }
  if (!have_device("yb_debug_conv_tf32")) return YB_ERR_NO_DEVICE;
  std::string d;
  float* ws = (float*)workspace;
  const size_t wsb = (size_t)workspace_bytes;
  int rc;
  if (pass == 0)
    rc = tf_conv_forward(x, w, bias, n, height, width, cin, cout, k, stride, k / 2, out, ws, wsb, 0, x_pitch, nullptr, &d);
  else if (pass == 1)
    rc = tf_conv_backward_data(dz, w, n, height, width, cin, cout, k, stride, k / 2, out, ws, wsb, 0, nullptr, &d);
  else
    rc = tf_conv_backward_weight(x, dz, n, height, width, cin, cout, k, stride, k / 2, out, ws, wsb, 0, x_pitch, &d);
  const cudaError_t ce = cudaDeviceSynchronize();
  if (!rc && ce != cudaSuccess) {
    set_error(std::string("yb_debug_conv_tf32: kernel failed: ") + cudaGetErrorString(ce));
    rc = YB_ERR_CUDA;
  }
  if (desc && desc_capacity > 0) snprintf(desc, (size_t)desc_capacity, "%s", d.c_str());
  return rc;
}

int32_t yb_debug_conv_tf32_eval(const float* x, int32_t x_pitch, const float* w, const float* gamma, const float* beta,
                                const float* running_mean, const float* running_var, int32_t n, int32_t height, int32_t width,
                                int32_t cin, int32_t cout, int32_t k, int32_t stride, int32_t act, const float* res, int32_t res_pitch,
                                float* out, int32_t out_pitch, int32_t out_coff, float* folded_w, float* folded_bias, char* desc,
                                int32_t desc_capacity) {
  if (!x || !w || !gamma || !beta || !running_mean || !running_var || !out || !folded_w || !folded_bias) {
    set_error("yb_debug_conv_tf32_eval: null argument");
    return YB_ERR_INVALID_ARG;
  }
  if (n <= 0 || height <= 0 || width <= 0 || cin <= 0 || cout <= 0 || x_pitch < 0 || res_pitch < 0 || out_pitch <= 0 || (act != 0 && act != 1)) {
    set_error("yb_debug_conv_tf32_eval: bad argument (extent, pitch or act)");
    return YB_ERR_INVALID_ARG;
  }
  if (!tf_shape_ok(cin, cout, k, stride, k / 2)) {
    set_error("yb_debug_conv_tf32_eval: shape not supported: channels must be multiples of 8, k in {1,3}, stride in {1,2}");
    return YB_ERR_SHAPE;
  }
  if (!have_device("yb_debug_conv_tf32_eval")) return YB_ERR_NO_DEVICE;
  TfFoldDesc fd{};
  fd.w = w; fd.gamma = gamma; fd.beta = beta; fd.rm = running_mean; fd.rv = running_var;
  fd.wf = folded_w; fd.bias = folded_bias;
  fd.cout = cout; fd.cin = cin; fd.taps = k * k;
  TfFoldDesc* dd = nullptr;
  YB_CUDA_CHECK(cudaMalloc((void**)&dd, sizeof(TfFoldDesc)));
  std::string d;
  int rc = cudaMemcpy(dd, &fd, sizeof(fd), cudaMemcpyHostToDevice) == cudaSuccess ? 0 : YB_ERR_CUDA;
  if (rc) set_error("yb_debug_conv_tf32_eval: descriptor copy failed");
  if (!rc) rc = tf_fold_all(dd, 1, tf_fold_chunks(fd), 0);
  if (!rc)
    rc = tf_conv_forward_eval(x, x_pitch ? x_pitch : cin, folded_w, folded_bias, n, height, width, cin, cout, k, stride, act, res,
                              res_pitch ? res_pitch : cout, out, out_pitch, out_coff, 0, &d);
  const cudaError_t ce = cudaDeviceSynchronize();
  if (!rc && ce != cudaSuccess) {
    set_error(std::string("yb_debug_conv_tf32_eval: kernel failed: ") + cudaGetErrorString(ce));
    rc = YB_ERR_CUDA;
  }
  cudaFree(dd);
  if (desc && desc_capacity > 0) snprintf(desc, (size_t)desc_capacity, "%s", d.c_str());
  return rc;
}

int32_t yb_stem_conv_forward_f32(const float* x, int32_t x_channels, const float* w, int32_t n, int32_t height, int32_t width,
                                 int32_t cout, float* z, void* stream) {
  if (!x || !w || !z || n <= 0 || height <= 0 || width <= 0 || cout <= 0) { set_error("yb_stem_conv_forward_f32: bad argument"); return YB_ERR_INVALID_ARG; }
  if (!have_device("yb_stem_conv_forward_f32")) return YB_ERR_NO_DEVICE;
  return stem3_forward(x, x_channels, w, n, height, width, cout, z, (cudaStream_t)stream);
}

int32_t yb_stem_conv_backward_weight_f32(const float* x, int32_t x_channels, const float* dz, int32_t n, int32_t height, int32_t width,
                                         int32_t cout, float* dw, void* workspace, int64_t workspace_bytes, void* stream) {
  if (!x || !dz || !dw || !workspace || n <= 0 || height <= 0 || width <= 0 || cout <= 0) { set_error("yb_stem_conv_backward_weight_f32: bad argument"); return YB_ERR_INVALID_ARG; }
  if (!have_device("yb_stem_conv_backward_weight_f32")) return YB_ERR_NO_DEVICE;
  return stem3_backward_weight(x, x_channels, dz, n, height, width, cout, dw, (float*)workspace, (size_t)workspace_bytes, (cudaStream_t)stream);
}

}  // extern "C"
