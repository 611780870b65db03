// Validation-side post-processing on the GPU (SURVEY.md section 8(f) row f3), batched over the images of a step:
//   * Metrics.box_iou            Utils/Metrics.cs:16-34   IoU = inter / (area1 + area2 - inter + eps), fp32
//   * match_predictions          Models/YoloBaseTaskModel.cs:377-446   the (detections x 10 IoU thresholds) true-positive
//                                 matrix that Detector.Val feeds to ap_per_class (Models/Detector.cs:103-120)
// The reference runs match_predictions per image on the host: nonzero -> argsort by IoU -> "unique by detection, then
// unique by label" with first occurrences found in a scalar loop of .item() calls.  What that procedure keeps is
//   best(d)  = the label with the highest IoU among the labels of d's class with IoU >= thr   (first unique: rows come
//              out ordered by detection index)
//   correct[d] = best(d) exists and d is the LOWEST detection index among { d' : best(d') == best(d) }   (second unique)
// which is what the kernel computes directly, one CTA per (image, threshold).
#include "common.cuh"

namespace yb {

__device__ __forceinline__ float box_iou_rn(float ax1, float ay1, float ax2, float ay2, float bx1, float by1, float bx2,
                                            float by2, float eps) {
  const float w = fmaxf(__fsub_rn(fminf(ax2, bx2), fmaxf(ax1, bx1)), 0.f);
  const float h = fmaxf(__fsub_rn(fminf(ay2, by2), fmaxf(ay1, by1)), 0.f);
  const float inter = __fmul_rn(w, h);
  const float a1 = __fmul_rn(__fsub_rn(ax2, ax1), __fsub_rn(ay2, ay1));
  const float a2 = __fmul_rn(__fsub_rn(bx2, bx1), __fsub_rn(by2, by1));
  return __fdiv_rn(inter, __fadd_rn(__fsub_rn(__fadd_rn(a1, a2), inter), eps));
}

__global__ void box_iou_kernel(const float* __restrict__ b1, int n, const float* __restrict__ b2, int m, float eps,
                               float* __restrict__ out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * m) return;
  const int i = idx / m, j = idx - i * m;
  out[idx] = box_iou_rn(b1[4 * i], b1[4 * i + 1], b1[4 * i + 2], b1[4 * i + 3], b2[4 * j], b2[4 * j + 1], b2[4 * j + 2],
                        b2[4 * j + 3], eps);
}

constexpr int MP_MAX_DET = 1024, MP_MAX_LABELS = 2048, MP_MAX_THR = 16;
struct MatchThr { float v[MP_MAX_THR]; };

__global__ void __launch_bounds__(256) match_predictions_kernel(const float* __restrict__ dets, const int* __restrict__ counts,
                                                                int max_det, int row_w, const float* __restrict__ labels,
                                                                int n_labels, MatchThr thr, int n_thr,
                                                                unsigned char* __restrict__ correct) {
  __shared__ int best[MP_MAX_DET];
  __shared__ int first_det[MP_MAX_LABELS];
  const int b = blockIdx.x, ti = blockIdx.y;
  const int n = min(counts[b], max_det);
  const float t = thr.v[ti];
  for (int l = threadIdx.x; l < n_labels; l += blockDim.x) first_det[l] = 0x7fffffff;
  __syncthreads();
  for (int d = threadIdx.x; d < n; d += blockDim.x) {
    const float* r = dets + ((size_t)b * max_det + d) * row_w;
    const float x1 = r[0], y1 = r[1], x2 = r[2], y2 = r[3], cls = r[5];
    int bl = -1;
    float bi = 0.f;
    for (int l = 0; l < n_labels; l++) {
      const float* g = labels + (size_t)l * 6;
      if ((int)g[0] != b || g[1] != cls) continue;  // iou * correct_class: other classes contribute 0 (< every threshold)
      const float iou = box_iou_rn(g[2], g[3], g[4], g[5], x1, y1, x2, y2, 1e-7f);
      if (iou >= t && (bl < 0 || iou > bi)) { bl = l; bi = iou; }
    }
    best[d] = bl;
    if (bl >= 0) atomicMin(&first_det[bl], d);
  }
  __syncthreads();
  for (int d = threadIdx.x; d < max_det; d += blockDim.x) {
    unsigned char c = 0;
    if (d < n && best[d] >= 0 && first_det[best[d]] == d) c = 1;
    correct[((size_t)b * max_det + d) * n_thr + ti] = c;
  }
}


// Metrics.mask_iou (Utils/Metrics.cs:120-125): iou[i][j] = inter / (sum(mask1[i]) + sum(mask2[j]) - inter + eps) with
// inter = max(mask1[i] . mask2[j], 0) over the n = H * W pixels of the flattened masks.  One block per (i, j): the three sums
// in one pass (warp shuffles, then the 8 warp partials in order).  Seg validation compares a few dozen masks per image
// (Models/Segmenter.cs:142): a latency-sized problem, not a GEMM worth tensor cores.
__global__ void __launch_bounds__(256) mask_iou_kernel(const float* __restrict__ m1, const float* __restrict__ m2, int n, float eps,
                                                       float* __restrict__ out, int M) {
  const int i = blockIdx.y, j = blockIdx.x;
  const float* a = m1 + (size_t)i * n;
  const float* b = m2 + (size_t)j * n;
  float inter = 0.f, sa = 0.f, sb = 0.f;
  for (int k = threadIdx.x; k < n; k += blockDim.x) {
    const float x = a[k], y = b[k];
    inter = fmaf(x, y, inter);
    sa += x;
    sb += y;
  }
  __shared__ float red[3][8];
  for (int o = 16; o; o >>= 1) {
    inter += __shfl_down_sync(0xffffffffu, inter, o);
    sa += __shfl_down_sync(0xffffffffu, sa, o);
    sb += __shfl_down_sync(0xffffffffu, sb, o);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { red[0][warp] = inter; red[1][warp] = sa; red[2][warp] = sb; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float t0 = 0.f, t1 = 0.f, t2 = 0.f;
    for (int w = 0; w < 8; w++) { t0 += red[0][w]; t1 += red[1][w]; t2 += red[2][w]; }
    t0 = fmaxf(t0, 0.f);
    out[(size_t)i * M + j] = __fdiv_rn(t0, __fadd_rn(__fsub_rn(__fadd_rn(t1, t2), t0), eps));
  }
}

// ---------------------------------------------------------------------------------------------------------------
// The per-batch tail of the trainer's validation pass (yb_trainer_val_batch, Models/Detector.cs:81-132) and its
// accumulators.  The running row count lives on the device, so a batch is queued without the host learning how many
// detections NMS kept; the host counts images and labels itself and passes the label offset in.
// ---------------------------------------------------------------------------------------------------------------

// staged target rows [image, cls, x, y, w, h] (normalised, sorted by image) -> labels [image, cls, x1, y1, x2, y2] in input
// pixels, in the reference's order: `bboxes * (w, h, w, h)` then `Ops.xywh2xyxy` (Ops.cs:68-81) - the same fp32 operations
// as oracle/ops.py; and the int32 class of every label into the accumulator
__global__ void val_labels_kernel(const float* __restrict__ rows, int n, float W, float H, float* __restrict__ labels,
                                  int* __restrict__ target_cls) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* r = rows + (size_t)i * 6;
  const float x = __fmul_rn(r[2], W), y = __fmul_rn(r[3], H), w = __fmul_rn(r[4], W), h = __fmul_rn(r[5], H);
  float* o = labels + (size_t)i * 6;
  o[0] = r[0];
  o[1] = r[1];
  o[2] = __fsub_rn(x, __fdiv_rn(w, 2.f));
  o[3] = __fsub_rn(y, __fdiv_rn(h, 2.f));
  o[4] = __fadd_rn(x, __fdiv_rn(w, 2.f));
  o[5] = __fadd_rn(y, __fdiv_rn(h, 2.f));
  target_cls[i] = (int)r[1];
}

// one CTA: the kept NMS rows of every image, in image order and score order within an image, appended at the device row
// counter; and `loss_items = loss_items + loss_detach` (Detector.cs:124).  A batch that would not fit raises the overflow
// flag and appends nothing.
__global__ void __launch_bounds__(1024) val_accumulate_kernel(const float* __restrict__ dets, const int* __restrict__ counts, int B,
                                                              const unsigned char* __restrict__ correct,
                                                              const float* __restrict__ loss_detach, ValAccum acc) {
  extern __shared__ int off[];  // B + 1 row offsets
  const int base = acc.state[0];
  if (threadIdx.x == 0) {
    int o = 0;
    for (int b = 0; b < B; b++) { off[b] = o; o += min(counts[b], VAL_MAX_DET); }
    off[B] = o;
  }
  if (threadIdx.x < 3) acc.loss[threadIdx.x] = __fadd_rn(acc.loss[threadIdx.x], loss_detach[threadIdx.x]);
  __syncthreads();
  const int total = off[B];
  if ((long long)base + total > acc.cap_rows) {
    if (threadIdx.x == 0) acc.state[1] = 1;
    return;
  }
  for (int i = threadIdx.x; i < total; i += blockDim.x) {
    int lo = 0, hi = B - 1;  // the image of output row i: the last b with off[b] <= i
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (off[mid] <= i) lo = mid; else hi = mid - 1;
    }
    const size_t src = (size_t)lo * VAL_MAX_DET + (i - off[lo]);
    const size_t dst = (size_t)base + i;
#pragma unroll
    for (int t = 0; t < VAL_T; t++) acc.tp[dst * VAL_T + t] = correct[src * VAL_T + t];
    acc.conf[dst] = dets[src * 6 + 4];
    acc.cls[dst] = (int)dets[src * 6 + 5];
  }
  __syncthreads();
  if (threadIdx.x == 0) acc.state[0] = base + total;
}

// one CTA: rows already in the accumulator layout (another rank's, gathered by the host) appended at the row counter, and
// their labels' classes at the host-known label offset
__global__ void __launch_bounds__(1024) val_append_rows_kernel(const unsigned char* __restrict__ tp, const float* __restrict__ conf,
                                                               const int* __restrict__ pred_cls, int n, const int* __restrict__ target_cls,
                                                               int m, long long label_off, ValAccum acc) {
  const int base = acc.state[0];
  for (int i = threadIdx.x; i < m; i += blockDim.x) acc.target_cls[label_off + i] = target_cls[i];
  if ((long long)base + n > acc.cap_rows) {
    if (threadIdx.x == 0) acc.state[1] = 1;
    return;
  }
  for (long long i = threadIdx.x; i < (long long)n * VAL_T; i += blockDim.x) acc.tp[(size_t)base * VAL_T + i] = tp[i];
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    acc.conf[(size_t)base + i] = conf[i];
    acc.cls[(size_t)base + i] = pred_cls[i];
  }
  __syncthreads();
  if (threadIdx.x == 0) acc.state[0] = base + n;
}

// Detector.Val's IoU vector torch.linspace(0.5, 0.95, 10) as ATen computes it in float32: the step rounded once, each value
// one rounding of start + step * i (first half) or end - step * (steps - 1 - i) (second half)
static MatchThr val_iouv() {
  MatchThr t;
  const float step = (0.95f - 0.5f) / 9.f;
  for (int i = 0; i < MP_MAX_THR; i++)
    t.v[i] = i >= VAL_T ? 2.f : (float)(i < 5 ? 0.5 + (double)step * i : (double)0.95f - (double)step * (VAL_T - 1 - i));
  return t;
}

int val_batch_launch(const float* pred, int B, int nc, int A, int H, int W, const float* rows, int n_labels, long long label_off,
                     const float* loss_detach, float* labels, float* dets, int* counts, unsigned char* correct, const ValAccum& acc,
                     cudaStream_t s) {
  static_assert(VAL_MAX_BATCH_LABELS == MP_MAX_LABELS, "the matching kernel's label limit");
  // these kernels follow ordinary launches (the loss, NMS and matching kernels), so they are launched the ordinary way
  val_labels_kernel<<<(n_labels + 255) / 256, 256, 0, s>>>(rows, n_labels, (float)W, (float)H, labels, acc.target_cls + label_off);
  YB_CUDA_CHECK(cudaGetLastError());
  // Ops.non_max_suppression(inference["boxes"], nc, conf_thres: 0.1, iou_thres: 0.7) with the defaults max_det 300,
  // max_nms 30000, max_wh 7680 (Detector.cs:97)
  if (int rc = nms_launch(pred, B, 4 + nc, A, nc, 0.1f, 0.7f, VAL_MAX_DET, 30000, 7680, dets, counts, nullptr, s)) return rc;
  match_predictions_kernel<<<dim3(B, VAL_T), 256, 0, s>>>(dets, counts, VAL_MAX_DET, 6, labels, n_labels, val_iouv(), VAL_T, correct);
  YB_CUDA_CHECK(cudaGetLastError());
  val_accumulate_kernel<<<1, 1024, (B + 1) * sizeof(int), s>>>(dets, counts, B, correct, loss_detach, acc);
  YB_CUDA_CHECK(cudaGetLastError());
  return YB_OK;
}

int val_append_launch(const unsigned char* tp, const float* conf, const int* pred_cls, int n, const int* target_cls, int m,
                      long long label_off, const ValAccum& acc, cudaStream_t s) {
  val_append_rows_kernel<<<1, 1024, 0, s>>>(tp, conf, pred_cls, n, target_cls, m, label_off, acc);
  YB_CUDA_CHECK(cudaGetLastError());
  return YB_OK;
}

}  // namespace yb

using namespace yb;

extern "C" {

int32_t yb_box_iou(const float* box1, int32_t n, const float* box2, int32_t m, float eps, float* out, void* stream) {
  if (n < 0 || m < 0 || ((n > 0 && m > 0) && (!box1 || !box2 || !out))) { set_error("yb_box_iou: bad argument"); return YB_ERR_INVALID_ARG; }
  if (n == 0 || m == 0) return YB_OK;
  box_iou_kernel<<<(n * m + 255) / 256, 256, 0, (cudaStream_t)stream>>>(box1, n, box2, m, eps, out);
  YB_CUDA_CHECK(cudaGetLastError());
  return YB_OK;
}

int32_t yb_mask_iou(const float* mask1, int32_t n1, const float* mask2, int32_t n2, int32_t pixels, float eps, float* out, void* stream) {
  if (n1 < 0 || n2 < 0 || pixels <= 0 || ((n1 > 0 && n2 > 0) && (!mask1 || !mask2 || !out))) { set_error("yb_mask_iou: bad argument"); return YB_ERR_INVALID_ARG; }
  if (n1 == 0 || n2 == 0) return YB_OK;
  if (n1 > 65535) { set_error("yb_mask_iou: at most 65535 rows in mask1"); return YB_ERR_INVALID_ARG; }
  mask_iou_kernel<<<dim3(n2, n1), 256, 0, (cudaStream_t)stream>>>(mask1, mask2, pixels, eps, out, n2);
  YB_CUDA_CHECK(cudaGetLastError());
  return YB_OK;
}

int32_t yb_match_predictions(const float* dets, const int32_t* counts, int32_t batch, int32_t max_det, int32_t row_width,
                             const float* labels, int32_t n_labels, const float* iou_thresholds_host, int32_t n_thresholds,
                             uint8_t* correct, void* stream) {
  if (!dets || !counts || !correct || !iou_thresholds_host || (n_labels > 0 && !labels)) { set_error("yb_match_predictions: null argument"); return YB_ERR_INVALID_ARG; }
  if (batch <= 0 || max_det <= 0 || max_det > MP_MAX_DET || row_width < 6 || n_labels < 0 || n_labels > MP_MAX_LABELS ||
      n_thresholds <= 0 || n_thresholds > MP_MAX_THR) {
    set_error("yb_match_predictions: need 0 < max_det <= 1024, row_width >= 6, n_labels <= 2048, 0 < n_thresholds <= 16");
    return YB_ERR_INVALID_ARG;
  }
  MatchThr t;
  for (int i = 0; i < MP_MAX_THR; i++) t.v[i] = i < n_thresholds ? iou_thresholds_host[i] : 2.f;
  match_predictions_kernel<<<dim3(batch, n_thresholds), 256, 0, (cudaStream_t)stream>>>(dets, counts, max_det, row_width, labels,
                                                                                      n_labels, t, n_thresholds, correct);
  YB_CUDA_CHECK(cudaGetLastError());
  return YB_OK;
}

}  // extern "C"
