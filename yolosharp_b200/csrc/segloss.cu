// The instance-mask term of v8SegmentationLoss on the GPU (SURVEY.md section 8(f) row f3), loss and gradients:
// `calculate_segmentation_loss` + `single_mask_loss` (Utils/Loss.cs:787-795, 806-861) as `v8SegmentationLoss.loss` uses them
// (:712-786, overlap_mask = true: the mask tensor holds instance index + 1 per pixel), fed by the assignment that
// yb_detection_loss already returns (fg, gt_idx) and the assigned boxes.
//
//   L = hyp_box / n_fg * sum over foreground anchors i of  [ sum over pixels p inside the box of i of BCE(m_i(p), g_i(p)) ] / (H W area_i)
//   m_i(p) = sum_k coef[b][k][i] * proto[b][k][p]          (einsum "in,nhw->ihw")
//   g_i(p) = masks[b][p] == gt_idx[b][i] + 1
//   box of i = target box / image size * mask size, cropped as Ops.crop_mask's tensor branch does (x1 <= col < x2, y1 <= row < y2, fp32),
//   area_i = (x2 - x1)(y2 - y1) of the box normalised to [0, 1]
// and, as the criterion returns loss * batch_size, the gradients are those of L * B:
//   dL/dm_i(p) = (sigmoid(m) - g) * s_i inside the box,  s_i = hyp_box * B / (n_fg H W area_i)
//   dcoef[b][k][i] = sum_p dm_i(p) proto[b][k][p]         one block per foreground anchor (fixed-order block reduction)
//   dproto[b][k][p] = sum_i dm_i(p) coef[b][k][i]         one thread per pixel walking the image's foreground anchors in
//                                                         anchor order (a gather: deterministic, no atomics)
// Work is HBM / L2 bound on `proto` (nm * H * W floats per image, re-read per foreground anchor from L2).
#include <algorithm>
#include <string>

#include "common.cuh"

namespace yb {

namespace {

constexpr int SG_MAX_NM = 64;

__device__ __forceinline__ float bce_logits(float x, float z) {  // max(x, 0) - x z + log(1 + exp(-|x|))
  return fmaxf(x, 0.f) - x * z + log1pf(expf(-fabsf(x)));
}

// one block per image: compact the foreground anchors (anchor order) with their boxes in mask pixels, area, instance id and
// coefficient vector; count them
__global__ void __launch_bounds__(1024) seg_compact_kernel(const unsigned char* __restrict__ fg, const int* __restrict__ gt_idx,
                                                           const float* __restrict__ tbox, const float* __restrict__ coef, int A, int nm,
                                                           int mh, int mw, float img_h, float img_w, int* __restrict__ list,
                                                           float* __restrict__ cbox, float* __restrict__ ccoef, int* __restrict__ counts,
                                                           int* __restrict__ total) {
  __shared__ int wsum[32];
  __shared__ int run;
  const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) run = 0;
  __syncthreads();
  for (int base = 0; base < A; base += 1024) {
    const int a = base + threadIdx.x;
    const int v = a < A && fg[(size_t)b * A + a] ? 1 : 0;
    int x = v;
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    int off = run;
    for (int w = 0; w < warp; w++) off += wsum[w];
    if (v) {
      const int j = off + x - 1;
      list[(size_t)b * A + j] = a;
      const float* t = tbox + ((size_t)b * A + a) * 4;
      // target_bboxes / imgsz[[1, 0, 1, 0]], then * (mask_w, mask_h, mask_w, mask_h) and the normalised area (Loss.cs:817-825)
      const float nx1 = __fdiv_rn(t[0], img_w), ny1 = __fdiv_rn(t[1], img_h), nx2 = __fdiv_rn(t[2], img_w), ny2 = __fdiv_rn(t[3], img_h);
      float* o = cbox + ((size_t)b * A + j) * 6;
      o[0] = __fmul_rn(nx1, (float)mw); o[1] = __fmul_rn(ny1, (float)mh); o[2] = __fmul_rn(nx2, (float)mw); o[3] = __fmul_rn(ny2, (float)mh);
      o[4] = __fmul_rn(__fsub_rn(nx2, nx1), __fsub_rn(ny2, ny1));
      o[5] = (float)(gt_idx[(size_t)b * A + a] + 1);
      for (int k = 0; k < nm; k++) ccoef[((size_t)b * A + j) * nm + k] = coef[((size_t)b * nm + k) * A + a];
    }
    __syncthreads();
    if (threadIdx.x == 0) { int s = 0; for (int w = 0; w < 32; w++) s += wsum[w]; run += s; }
    __syncthreads();
  }
  if (threadIdx.x == 0) { counts[b] = run; atomicAdd(total, run); }
}

// block (foreground rank j, image b): BCE over the box, d/dcoef
template <int NM>  // register arrays of NM coefficients: 32 (the reference's nm) or 64
__global__ void __launch_bounds__(256) seg_anchor_kernel(const int* __restrict__ list, const float* __restrict__ cbox,
                                                         const float* __restrict__ ccoef, const int* __restrict__ counts,
                                                         const int* __restrict__ total, const float* __restrict__ masks,
                                                         const float* __restrict__ proto, int B, int A, int nm, int mh, int mw, float hyp_box,
                                                         float* __restrict__ lossbuf, float* __restrict__ gcoef) {
  const int j = blockIdx.x, b = blockIdx.y;
  if (j >= counts[b]) return;
  __shared__ float sc[NM];
  __shared__ float red[8][NM + 1];
  const float* bx = cbox + ((size_t)b * A + j) * 6;
  const float x1 = bx[0], y1 = bx[1], x2 = bx[2], y2 = bx[3], area = bx[4], inst = bx[5];
  for (int k = threadIdx.x; k < nm; k += blockDim.x) sc[k] = ccoef[((size_t)b * A + j) * nm + k];
  __syncthreads();
  const int hw = mh * mw;
  const float* P = proto + (size_t)b * nm * hw;
  const float* M = masks + (size_t)b * hw;
  // rows / columns that can pass the fp32 comparisons of crop_mask (the exact test is repeated per pixel)
  const int c0 = max(0, (int)floorf(x1)), c1 = min(mw, (int)ceilf(x2) + 1), r0 = max(0, (int)floorf(y1)), r1 = min(mh, (int)ceilf(y2) + 1);
  const int bw = max(c1 - c0, 0), bh = max(r1 - r0, 0);
  const float s = __fdiv_rn(hyp_box * (float)B, (float)*total * (float)hw * area);  // d(L * B) / d(sum of BCE of this anchor)
  float lsum = 0.f;
  float dk[NM];
#pragma unroll
  for (int k = 0; k < NM; k++) dk[k] = 0.f;
  for (int i = threadIdx.x; i < bw * bh; i += blockDim.x) {
    const int r = r0 + i / bw, c = c0 + i % bw;
    if (!((float)c >= x1 && (float)c < x2 && (float)r >= y1 && (float)r < y2)) continue;
    const int p = r * mw + c;
    float pk[NM];
    float m = 0.f;
#pragma unroll
    for (int k = 0; k < NM; k++) {
      pk[k] = k < nm ? P[(size_t)k * hw + p] : 0.f;
      if (k < nm) m = fmaf(sc[k], pk[k], m);
    }
    const float g = M[p] == inst ? 1.f : 0.f;
    lsum += bce_logits(m, g);
    const float dm = (1.f / (1.f + expf(-m)) - g) * s;
#pragma unroll
    for (int k = 0; k < NM; k++) dk[k] = fmaf(dm, pk[k], dk[k]);
  }
  // block reduction in a fixed order: lanes by shuffle, warps through shared memory
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int o = 16; o; o >>= 1) lsum += __shfl_down_sync(0xffffffffu, lsum, o);
#pragma unroll
  for (int k = 0; k < NM; k++) {
    if (k < nm) {
      float v = dk[k];
      for (int o = 16; o; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
      if (lane == 0) red[warp][k] = v;
    }
  }
  if (lane == 0) red[warp][NM] = lsum;
  __syncthreads();
  const int a = list[(size_t)b * A + j];
  for (int k = threadIdx.x; k <= nm; k += blockDim.x) {
    const int kk = k < nm ? k : NM;
    float v = 0.f;
    for (int w = 0; w < 8; w++) v += red[w][kk];
    if (k < nm) gcoef[((size_t)b * nm + k) * A + a] = v;
    else lossbuf[(size_t)b * A + j] = __fdiv_rn(__fdiv_rn(v, (float)hw), area);  // crop(loss).mean((1, 2)) / area
  }
}

// thread (pixel p, image b): d/dproto as a gather over the image's foreground anchors, in anchor order
template <int NM>
__global__ void __launch_bounds__(128) seg_proto_kernel(const float* __restrict__ cbox, const float* __restrict__ ccoef,
                                                        const int* __restrict__ counts, const int* __restrict__ total,
                                                        const float* __restrict__ masks, const float* __restrict__ proto, int B, int A, int nm,
                                                        int mh, int mw, float hyp_box, float* __restrict__ gproto) {
  const int hw = mh * mw, b = blockIdx.y;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = counts[b];
  __shared__ float sb[32][6];
  __shared__ float sc[32][NM];
  const bool on = p < hw;
  const int r = on ? p / mw : 0, c = on ? p - r * mw : 0;
  float pv[NM], acc[NM];
#pragma unroll
  for (int k = 0; k < NM; k++) {
    pv[k] = (on && k < nm) ? proto[((size_t)b * nm + k) * hw + p] : 0.f;
    acc[k] = 0.f;
  }
  const float mval = on ? masks[(size_t)b * hw + p] : -1.f;
  const float tot = (float)*total;
  for (int j0 = 0; j0 < n; j0 += 32) {  // 32 anchors at a time through shared memory
    __syncthreads();
    const int cnt = min(32, n - j0);
    for (int i = threadIdx.x; i < cnt * 6; i += blockDim.x) sb[i / 6][i % 6] = cbox[((size_t)b * A + j0) * 6 + i];
    for (int i = threadIdx.x; i < cnt * nm; i += blockDim.x) sc[i / nm][i % nm] = ccoef[((size_t)b * A + j0) * nm + i];
    __syncthreads();
    if (!on) continue;
    for (int jj = 0; jj < cnt; jj++) {
      if (!((float)c >= sb[jj][0] && (float)c < sb[jj][2] && (float)r >= sb[jj][1] && (float)r < sb[jj][3])) continue;
      float m = 0.f;
#pragma unroll
      for (int k = 0; k < NM; k++)
        if (k < nm) m = fmaf(sc[jj][k], pv[k], m);
      const float g = mval == sb[jj][5] ? 1.f : 0.f;
      const float s = __fdiv_rn(hyp_box * (float)B, tot * (float)hw * sb[jj][4]);
      const float dm = (1.f / (1.f + expf(-m)) - g) * s;
#pragma unroll
      for (int k = 0; k < NM; k++)
        if (k < nm) acc[k] = fmaf(dm, sc[jj][k], acc[k]);
    }
  }
  if (!on) return;
#pragma unroll
  for (int k = 0; k < NM; k++)
    if (k < nm) gproto[((size_t)b * nm + k) * hw + p] = acc[k];
}

// one block: loss item = hyp_box * (sum of the per-anchor terms in (image, anchor) order) / n_fg
__global__ void __launch_bounds__(256) seg_item_kernel(const float* __restrict__ lossbuf, const int* __restrict__ counts,
                                                       const int* __restrict__ total, int B, int A, float hyp_box, float* __restrict__ item) {
  __shared__ float red[256];
  float acc = 0.f;
  for (int b = 0; b < B; b++)
    for (int j = threadIdx.x; j < counts[b]; j += 256) acc += lossbuf[(size_t)b * A + j];
  red[threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 256; i++) t += red[i];
    item[0] = *total > 0 ? __fmul_rn(__fdiv_rn(t, (float)*total), hyp_box) : 0.f;
  }
}

}  // namespace

}  // namespace yb

using namespace yb;

extern "C" int32_t yb_segmentation_loss(const uint8_t* fg, const int32_t* gt_idx, const float* target_bboxes, const float* masks,
                                        const float* proto, const float* mask_coefficient, int32_t batch, int32_t anchors, int32_t nm,
                                        int32_t mask_h, int32_t mask_w, float img_h, float img_w, float hyp_box, float* loss_item,
                                        float* grad_proto, float* grad_coefficient, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (!fg || !gt_idx || !target_bboxes || !masks || !proto || !mask_coefficient || !loss_item || !grad_proto || !grad_coefficient) {
    set_error("yb_segmentation_loss: null argument");
    return YB_ERR_INVALID_ARG;
  }
  if (batch <= 0 || anchors <= 0 || nm <= 0 || nm > SG_MAX_NM || mask_h <= 0 || mask_w <= 0 || img_h <= 0 || img_w <= 0 ||
      (long long)mask_h * mask_w > (1 << 24)) {
    set_error("yb_segmentation_loss: need 0 < nm <= 64 and positive sizes");
    return YB_ERR_SHAPE;
  }
  if (!have_device("yb_segmentation_loss")) return YB_ERR_NO_DEVICE;
  const size_t BA = (size_t)batch * anchors;
  // scratch: list (int) | counts (int) | total (int) | cbox (6 f) | ccoef (nm f) | lossbuf (f)
  const size_t bytes = BA * 4 + (size_t)batch * 4 + 16 + BA * 6 * 4 + BA * nm * 4 + BA * 4 + 64;
  char* scratch = nullptr;
  YB_CUDA_CHECK(cudaMallocAsync((void**)&scratch, bytes, s));
  int* list = reinterpret_cast<int*>(scratch);
  int* counts = list + BA;
  int* total = counts + batch;
  float* cbox = reinterpret_cast<float*>(scratch + ((BA * 4 + (size_t)batch * 4 + 4 + 15) / 16) * 16);
  float* ccoef = cbox + BA * 6;
  float* lossbuf = ccoef + BA * nm;
  const int hw = mask_h * mask_w;
  cudaError_t ce = cudaMemsetAsync(total, 0, 4, s);
  if (ce == cudaSuccess) ce = cudaMemsetAsync(grad_coefficient, 0, (size_t)batch * nm * anchors * sizeof(float), s);
  if (ce == cudaSuccess) {
    seg_compact_kernel<<<batch, 1024, 0, s>>>(fg, gt_idx, target_bboxes, mask_coefficient, anchors, nm, mask_h, mask_w, img_h, img_w, list, cbox,
                                              ccoef, counts, total);
    if (nm <= 32) {
      seg_anchor_kernel<32><<<dim3(anchors, batch), 256, 0, s>>>(list, cbox, ccoef, counts, total, masks, proto, batch, anchors, nm, mask_h,
                                                                 mask_w, hyp_box, lossbuf, grad_coefficient);
      seg_proto_kernel<32><<<dim3((hw + 127) / 128, batch), 128, 0, s>>>(cbox, ccoef, counts, total, masks, proto, batch, anchors, nm, mask_h,
                                                                         mask_w, hyp_box, grad_proto);
    } else {
      seg_anchor_kernel<64><<<dim3(anchors, batch), 256, 0, s>>>(list, cbox, ccoef, counts, total, masks, proto, batch, anchors, nm, mask_h,
                                                                 mask_w, hyp_box, lossbuf, grad_coefficient);
      seg_proto_kernel<64><<<dim3((hw + 127) / 128, batch), 128, 0, s>>>(cbox, ccoef, counts, total, masks, proto, batch, anchors, nm, mask_h,
                                                                         mask_w, hyp_box, grad_proto);
    }
    seg_item_kernel<<<1, 256, 0, s>>>(lossbuf, counts, total, batch, anchors, hyp_box, loss_item);
    ce = cudaGetLastError();
  }
  cudaFreeAsync(scratch, s);
  if (ce != cudaSuccess) { set_error(std::string("yb_segmentation_loss: ") + cudaGetErrorString(ce)); return YB_ERR_CUDA; }
  return YB_OK;
}
