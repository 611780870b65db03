// Metrics.ap_per_class on the GPU (SURVEY.md section 8(f) row f3): the reduction that `Detector.Val` runs once per validation
// pass over ALL detections of the set (Utils/Metrics.cs:308-384, with compute_ap :395-421, interp :424-468, smooth :475-487).
// HBM / latency-bound integer and fp32 work: two key sorts, segmented scans, binary searches.
//
//   1. order by confidence  : bitonic sort of 64-bit keys (~ordered(conf) << 32 | index): descending confidence, equal
//                             confidences in input order.  The reference calls torch.argsort(-conf) (unstable): wherever
//                             it has ties its result is unspecified; this kernel (and oracle/val.py) use the stable order.
//   2. class-major order    : second sort of (class << 32 | rank): every class becomes one contiguous segment, still in
//                             confidence order - the reference's boolean mask `pred_cls == c` per class
//   3. per (class, IoU thr) : cumulative TP / FP -> recall, precision (fp32, as the reference's int64 / float divisions)
//                             and the precision envelope (reverse running max, compute_ap)
//   4. per (class, IoU thr) : 101-point interpolated AP (the reference's own `interp`: left value 0, right value fp[-1])
//   5. per class            : precision / recall curves over 1000 confidence points, precision-at-recall values (thr 0)
//   6. one block            : F1 curves, their class mean smoothed by a 201-tap box filter (both pads repeat y[0], as
//                             the reference does), arg-max, and p / r / f1 / tp / fp at that index
// Precondition (true for match_predictions' output): per class and threshold the number of true positives does not
// exceed the number of labels, so recall <= 1 and compute_ap's `mrec` is already sorted.
#include <algorithm>
#include <cstdlib>
#include <vector>

#include "common.cuh"

namespace yb {

namespace {

constexpr int AP_PTS = 1000, AP_COCO = 101, AP_MAX_T = 16, AP_MAX_CLASSES = 4096;

__device__ __forceinline__ unsigned ord_key(float v) {
  const unsigned u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);  // ascending integer order == ascending float order
}

// ---- bitonic sort of 64-bit keys in global memory (n2 = power of two) ----
__global__ void bitonic_global_kernel(unsigned long long* __restrict__ k, int j, int kk, int n2) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n2) return;
  const int ixj = i ^ j;
  if (ixj > i) {
    const unsigned long long a = k[i], b = k[ixj];
    if ((a > b) == ((i & kk) == 0)) { k[i] = b; k[ixj] = a; }
  }
}
// all steps with j < 1024 of stage kk (or, first = 1, all stages kk <= 1024) inside one 1024-key chunk of shared memory
__global__ void __launch_bounds__(512) bitonic_local_kernel(unsigned long long* __restrict__ k, int kk, int first, int n2) {
  __shared__ unsigned long long s[1024];
  const int base = blockIdx.x * 1024;
  for (int t = threadIdx.x; t < 1024; t += 512) s[t] = base + t < n2 ? k[base + t] : ~0ull;
  __syncthreads();
  const int k_lo = first ? 2 : kk, k_hi = first ? min(1024, n2) : kk;
  for (int ks = k_lo; ks <= k_hi; ks <<= 1) {
    for (int j = min(ks >> 1, 512); j > 0; j >>= 1) {
      for (int t = threadIdx.x; t < 1024; t += 512) {
        const int ixj = t ^ j;
        if (ixj > t) {
          const unsigned long long a = s[t], b = s[ixj];
          if ((a > b) == (((base + t) & ks) == 0)) { s[t] = b; s[ixj] = a; }
        }
      }
      __syncthreads();
    }
  }
  for (int t = threadIdx.x; t < 1024; t += 512)
    if (base + t < n2) k[base + t] = s[t];
}
int sort_keys(unsigned long long* keys, int n2, cudaStream_t s) {
  const int chunks = (n2 + 1023) / 1024;
  bitonic_local_kernel<<<chunks, 512, 0, s>>>(keys, 0, 1, n2);
  for (int kk = 2048; kk <= n2; kk <<= 1) {
    for (int j = kk >> 1; j >= 1024; j >>= 1) bitonic_global_kernel<<<(n2 + 255) / 256, 256, 0, s>>>(keys, j, kk, n2);
    bitonic_local_kernel<<<chunks, 512, 0, s>>>(keys, kk, 0, n2);
  }
  YB_CUDA_CHECK(cudaGetLastError());
  return YB_OK;
}

__global__ void conf_keys_kernel(const float* __restrict__ conf, int n, int n2, unsigned long long* __restrict__ keys) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n2) return;
  keys[i] = i < n ? ((unsigned long long)(~ord_key(conf[i])) << 32) | (unsigned)i : ~0ull;
}
// rank r of the confidence order -> (class << 32 | r); histograms of the predicted and the target classes
__global__ void class_keys_kernel(const unsigned long long* __restrict__ k1, const int* __restrict__ pred_cls, int n, int n2,
                                  int max_classes, unsigned long long* __restrict__ k2, int* __restrict__ n_pred) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n2) return;
  if (r >= n) { k2[r] = ~0ull; return; }
  const int c = pred_cls[(unsigned)(k1[r] & 0xffffffffu)];
  if (c < 0 || c >= max_classes) { k2[r] = ~0ull - 1; return; }  // a class no label can have: sorted behind every segment
  k2[r] = ((unsigned long long)c << 32) | (unsigned)r;
  atomicAdd(&n_pred[c], 1);
}
__global__ void target_hist_kernel(const int* __restrict__ target_cls, int m, int max_classes, int* __restrict__ n_lab) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m && target_cls[i] >= 0 && target_cls[i] < max_classes) atomicAdd(&n_lab[target_cls[i]], 1);
}
// one block: segment starts (exclusive scan of n_pred in class order) and the sorted list of classes that have labels
__global__ void __launch_bounds__(1024) classes_kernel(const int* __restrict__ n_pred, const int* __restrict__ n_lab, int max_classes,
                                                       int* __restrict__ seg_start, int* __restrict__ uniq, int* __restrict__ n_uniq) {
  __shared__ int sp[AP_MAX_CLASSES], su[AP_MAX_CLASSES];
  for (int c = threadIdx.x; c < max_classes; c += blockDim.x) { sp[c] = n_pred[c]; su[c] = n_lab[c] > 0 ? 1 : 0; }
  __syncthreads();
  if (threadIdx.x == 0) {  // <= 4096 classes, once per validation pass
    int a = 0, u = 0;
    for (int c = 0; c < max_classes; c++) {
      seg_start[c] = a;
      a += sp[c];
      if (su[c]) uniq[u++] = c;
    }
    *n_uniq = u;
  }
}

// class-major gather: confidence and TP row of every sorted detection
__global__ void gather_kernel(const unsigned long long* __restrict__ k1, const unsigned long long* __restrict__ k2, const float* __restrict__ conf,
                              const unsigned char* __restrict__ tp, int n, int T, float* __restrict__ cconf,
                              unsigned char* __restrict__ ctp) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n) return;
  const unsigned long long key = k2[q];
  if (key >= ~0ull - 1) return;  // out-of-range class
  const unsigned idx = (unsigned)(k1[(unsigned)(key & 0xffffffffu)] & 0xffffffffu);
  cconf[q] = conf[idx];
  for (int j = 0; j < T; j++) ctp[(size_t)j * n + q] = tp[(size_t)idx * T + j] ? 1 : 0;
}

// block (class index ci, threshold j): cumulative TP -> recall / precision, then the precision envelope from the right
__global__ void __launch_bounds__(1024) pr_kernel(const int* __restrict__ uniq, const int* __restrict__ n_uniq, const int* __restrict__ seg_start,
                                                  const int* __restrict__ n_pred, const int* __restrict__ n_lab,
                                                  const unsigned char* __restrict__ ctp, int n, int ne, float* __restrict__ rec,
                                                  float* __restrict__ prec, float* __restrict__ env) {
  const int ci = blockIdx.x, j = blockIdx.y;
  if (ci >= *n_uniq) return;
  const int c = uniq[ci], s0 = seg_start[c], np = n_pred[c], nl = n_lab[c];
  if (np == 0 || nl == 0) return;
  __shared__ int wsum[32];
  __shared__ int run;
  __shared__ float wmax[32];
  __shared__ float runmax;
  if (threadIdx.x == 0) { run = 0; runmax = 0.f; }
  __syncthreads();
  const unsigned char* t = ctp + (size_t)j * n + s0;
  // rec / prec / env rows have ne = n + 2 * max_classes entries: the segment of class c starts at s0 + 2 c and carries
  // compute_ap's sentinels around its np values (mrec = [0, recall, 1], mpre = [1, envelope, 0])
  float* R = rec + (size_t)j * ne + s0 + 2 * c + 1;
  float* P = prec + (size_t)j * ne + s0 + 2 * c + 1;
  float* E = env + (size_t)j * ne + s0 + 2 * c + 1;
  if (threadIdx.x == 0) { R[-1] = 0.f; R[np] = 1.f; E[-1] = 1.f; E[np] = 0.f; }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int base = 0; base < np; base += 1024) {
    const int i = base + threadIdx.x;
    const int v = i < np ? t[i] : 0;
    int x = v;
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    int off = run;
    for (int w = 0; w < warp; w++) off += wsum[w];
    const int tpc = off + x;
    if (i < np) {
      R[i] = __fdiv_rn((float)tpc, (float)nl);        // tpc / (n_l + eps): eps = 1e-16f vanishes in fp32
      P[i] = __fdiv_rn((float)tpc, (float)(i + 1));   // tpc / (tpc + fpc)
    }
    __syncthreads();
    if (threadIdx.x == 0) { int a = 0; for (int w = 0; w < 32; w++) a += wsum[w]; run += a; }
    __syncthreads();
  }
  // envelope: mpre.flip(0).cummax(0).flip(0) over [1, precision..., 0] restricted to the precision entries = suffix max
  for (int hi = np; hi > 0; hi -= 1024) {
    const int i = hi - 1 - (int)threadIdx.x;  // thread 0 takes the right-most element of the chunk
    float x = i >= 0 ? P[i] : 0.f;
    for (int o = 1; o < 32; o <<= 1) { const float y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x = fmaxf(x, y); }
    if (lane == 31) wmax[warp] = x;
    __syncthreads();
    float m = runmax;
    for (int w = 0; w < warp; w++) m = fmaxf(m, wmax[w]);
    x = fmaxf(x, m);
    if (i >= 0) E[i] = x;
    __syncthreads();
    if (threadIdx.x == 0) { float a = runmax; for (int w = 0; w < 32; w++) a = fmaxf(a, wmax[w]); runmax = a; }
    __syncthreads();
  }
}

// the reference's interp (Metrics.cs:424-468) over a sorted abscissa accessed through xp(i), values fp(i), L points
template <typename FX, typename FY>
__device__ __forceinline__ float interp_ref(float x, int L, FX xp, FY fp, float left) {
  const float x_first = xp(0), x_last = xp(L - 1);
  if (x <= x_first) return left;          // written last in the reference: wins over the right-hand rule
  if (x >= x_last) return fp(L - 1);
  int lo = 0, hi = L;                      // searchsorted (left): first index with xp >= x
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (xp(mid) < x) lo = mid + 1; else hi = mid;
  }
  int k = lo - 1;
  k = max(0, min(k, L - 2));
  const float x0 = xp(k), x1 = xp(k + 1), y0 = fp(k), y1 = fp(k + 1);
  const float t = __fdiv_rn(__fsub_rn(x, x0), __fsub_rn(x1, x0));
  return __fadd_rn(y0, __fmul_rn(t, __fsub_rn(y1, y0)));
}

// block (ci, j): compute_ap - 101-point interpolation of (mrec, mpre) and the trapezoid
__global__ void __launch_bounds__(128) ap_kernel(const int* __restrict__ uniq, const int* __restrict__ n_uniq, const int* __restrict__ seg_start,
                                                 const int* __restrict__ n_pred, const int* __restrict__ n_lab, const float* __restrict__ rec,
                                                 const float* __restrict__ env, int ne, int T, const float* __restrict__ x101,
                                                 float* __restrict__ ap) {
  const int ci = blockIdx.x, j = blockIdx.y;
  if (ci >= *n_uniq) return;
  const int c = uniq[ci], s0 = seg_start[c], np = n_pred[c], nl = n_lab[c];
  if (np == 0 || nl == 0) return;  // ap stays 0
  __shared__ float y[AP_COCO];
  const float* R = rec + (size_t)j * ne + s0 + 2 * c;   // mrec, sentinels included
  const float* E = env + (size_t)j * ne + s0 + 2 * c;   // mpre
  const int L = np + 2;
  auto xp = [&](int i) { return R[i]; };
  auto fp = [&](int i) { return E[i]; };
  for (int k = threadIdx.x; k < AP_COCO; k += blockDim.x) y[k] = interp_ref(x101[k], L, xp, fp, 0.f);
  __syncthreads();
  if (threadIdx.x == 0) {
    float acc = 0.f;  // torch.trapezoid: sum((y[1:] + y[:-1]) * dx) / 2
    for (int k = 0; k + 1 < AP_COCO; k++) acc = __fadd_rn(acc, __fmul_rn(__fadd_rn(y[k + 1], y[k]), __fsub_rn(x101[k + 1], x101[k])));
    ap[(size_t)ci * T + j] = __fmul_rn(acc, 0.5f);
  }
}

// block ci: r_curve / p_curve over the 1000 confidence points (threshold 0) and the precision-at-recall row
__global__ void __launch_bounds__(1024) curves_kernel(const int* __restrict__ uniq, const int* __restrict__ n_uniq, const int* __restrict__ seg_start,
                                                      const int* __restrict__ n_pred, const int* __restrict__ n_lab,
                                                      const float* __restrict__ cconf, const float* __restrict__ rec,
                                                      const float* __restrict__ prec, const float* __restrict__ env,
                                                      int ne, const float* __restrict__ x1000, float* __restrict__ p_curve,
                                                      float* __restrict__ r_curve, float* __restrict__ prec_values,
                                                      const int* __restrict__ prec_row) {
  const int ci = blockIdx.x;
  if (ci >= *n_uniq) return;
  const int c = uniq[ci], s0 = seg_start[c], np = n_pred[c], nl = n_lab[c];
  if (np == 0 || nl == 0) return;  // rows stay 0
  (void)ne;
  const float* C = cconf + s0;
  const float* R = rec + s0 + 2 * c + 1;   // threshold 0; R[-1], R[np] are compute_ap's sentinels
  const float* P = prec + s0 + 2 * c + 1;
  const float* E = env + s0 + 2 * c + 1;
  auto xneg = [&](int i) { return -C[i]; };
  const int L = np + 2;
  auto mrec = [&](int i) { return R[i - 1]; };
  auto mpre = [&](int i) { return E[i - 1]; };
  for (int k = threadIdx.x; k < AP_PTS; k += blockDim.x) {
    const float xq = -x1000[k];
    r_curve[(size_t)ci * AP_PTS + k] = interp_ref(xq, np, xneg, [&](int i) { return R[i]; }, 0.f);
    p_curve[(size_t)ci * AP_PTS + k] = interp_ref(xq, np, xneg, [&](int i) { return P[i]; }, 1.f);
    prec_values[(size_t)prec_row[ci] * AP_PTS + k] = interp_ref(x1000[k], L, mrec, mpre, 0.f);
  }
}
// which row of prec_values a class writes (the reference appends one row per class that has predictions AND labels)
__global__ void prec_rows_kernel(const int* __restrict__ uniq, const int* __restrict__ n_uniq, const int* __restrict__ n_pred,
                                 const int* __restrict__ n_lab, int* __restrict__ prec_row, int* __restrict__ n_prec) {
  if (threadIdx.x || blockIdx.x) return;
  int r = 0;
  for (int ci = 0; ci < *n_uniq; ci++) {
    const int c = uniq[ci];
    prec_row[ci] = r;
    if (n_pred[c] > 0 && n_lab[c] > 0) r++;
  }
  *n_prec = r;
}

// one block: f1 curves, smoothed class mean, arg-max, statistics at the best point
__global__ void __launch_bounds__(1024) f1_kernel(const int* __restrict__ uniq, const int* __restrict__ n_uniq, const int* __restrict__ n_lab,
                                                  const float* __restrict__ p_curve, const float* __restrict__ r_curve,
                                                  float* __restrict__ f1_curve, float eps, float* __restrict__ p, float* __restrict__ r,
                                                  float* __restrict__ f1, float* __restrict__ tp, float* __restrict__ fp,
                                                  int* __restrict__ best_out) {
  __shared__ float mean[AP_PTS], sm[AP_PTS];
  __shared__ int best;
  const int nc = *n_uniq;
  for (int k = threadIdx.x; k < AP_PTS; k += blockDim.x) {
    float acc = 0.f;
    for (int ci = 0; ci < nc; ci++) {
      const float pv = p_curve[(size_t)ci * AP_PTS + k], rv = r_curve[(size_t)ci * AP_PTS + k];
      const float f = __fdiv_rn(__fmul_rn(__fmul_rn(2.f, pv), rv), __fadd_rn(__fadd_rn(pv, rv), eps));
      f1_curve[(size_t)ci * AP_PTS + k] = f;
      acc = __fadd_rn(acc, f);
    }
    mean[k] = nc > 0 ? __fdiv_rn(acc, (float)nc) : 0.f;
  }
  __syncthreads();
  // smooth(y, 0.1): nf = 201, both pads repeat y[0] (Metrics.cs:478-480), valid convolution with 1 / nf
  constexpr int NF = (int)(AP_PTS * 0.1f * 2) / 2 * 2 + 1, HALF = NF / 2;
  const float wgt = 1.f / (float)NF;
  for (int k = threadIdx.x; k < AP_PTS; k += blockDim.x) {
    float acc = 0.f;
    for (int t = 0; t < NF; t++) {
      const int src = k + t - HALF;  // index into y; outside -> y[0]
      acc = fmaf((src >= 0 && src < AP_PTS) ? mean[src] : mean[0], wgt, acc);
    }
    sm[k] = acc;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int b = 0;
    for (int k = 1; k < AP_PTS; k++) if (sm[k] > sm[b]) b = k;  // first maximum
    best = b;
    *best_out = b;
  }
  __syncthreads();
  for (int ci = threadIdx.x; ci < nc; ci += blockDim.x) {
    const float pv = p_curve[(size_t)ci * AP_PTS + best], rv = r_curve[(size_t)ci * AP_PTS + best];
    p[ci] = pv;
    r[ci] = rv;
    f1[ci] = f1_curve[(size_t)ci * AP_PTS + best];
    const float t = rintf(__fmul_rn(rv, (float)n_lab[uniq[ci]]));  // (r * nt).round(): half to even
    tp[ci] = t;
    fp[ci] = rintf(__fsub_rn(__fdiv_rn(t, __fadd_rn(pv, eps)), t));
  }
}

// torch.linspace(0, 1, steps) as ATen's CPU kernel computes it: a float32 step, symmetric about the middle, each value
// one rounding of start + step * i / end - step * (steps - 1 - i) (product and sum carried exactly: double here);
// tests/test_metrics.py compares with torch.linspace bit for bit
void linspace01(int steps, std::vector<float>& out) {
  out.resize(steps);
  const double step = (double)(1.0f / (float)(steps - 1));
  const int half = steps / 2;
  for (int i = 0; i < steps; i++) out[i] = (float)(i < half ? step * (double)i : 1.0 - step * (double)(steps - i - 1));
}

}  // namespace

}  // namespace yb

using namespace yb;

extern "C" {

int32_t yb_linspace01(int32_t steps, float* out_host) {
  if (steps < 2 || !out_host) { set_error("yb_linspace01: bad argument"); return YB_ERR_INVALID_ARG; }
  std::vector<float> v;
  linspace01(steps, v);
  std::copy(v.begin(), v.end(), out_host);
  return YB_OK;
}

int32_t yb_ap_per_class(const uint8_t* tp, const float* conf, const int32_t* pred_cls, int32_t n, int32_t n_thresholds,
                        const int32_t* target_cls, int32_t m, int32_t max_classes, int32_t* unique_classes, int32_t* counts_host,
                        float* ap, float* p_curve, float* r_curve, float* f1_curve, float* prec_values, float* p, float* r, float* f1,
                        float* tp_out, float* fp_out, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (n < 0 || m < 0 || n_thresholds <= 0 || n_thresholds > AP_MAX_T || max_classes <= 0 || max_classes > AP_MAX_CLASSES) {
    set_error("yb_ap_per_class: need 0 < n_thresholds <= 16, 0 < max_classes <= 4096");
    return YB_ERR_INVALID_ARG;
  }
  if ((n > 0 && (!tp || !conf || !pred_cls)) || (m > 0 && !target_cls) || !unique_classes || !counts_host || !ap || !p_curve || !r_curve ||
      !f1_curve || !prec_values || !p || !r || !f1 || !tp_out || !fp_out) {
    set_error("yb_ap_per_class: null argument");
    return YB_ERR_INVALID_ARG;
  }
  if (!have_device("yb_ap_per_class")) return YB_ERR_NO_DEVICE;
  const int T = n_thresholds;
  int n2 = 1024;
  while (n2 < n) n2 <<= 1;
  const size_t nn = (size_t)std::max(n, 1);
  const int ne = n + 2 * max_classes;  // row length of rec / prec / env (sentinels around every class segment)
  // scratch: k1 | k2 | rec | prec | env | cconf | x1000 | x101 | ints | ctp
  const size_t f_count = (size_t)3 * ne * T + nn + AP_PTS + AP_COCO;
  const size_t i_count = (size_t)4 * max_classes + 4;
  const size_t bytes = (size_t)2 * n2 * 8 + f_count * 4 + i_count * 4 + nn * T + 64;
  char* scratch = nullptr;
  YB_CUDA_CHECK(cudaMallocAsync((void**)&scratch, bytes, s));
  unsigned long long* k1 = reinterpret_cast<unsigned long long*>(scratch);
  unsigned long long* k2 = k1 + n2;
  float* rec = reinterpret_cast<float*>(k2 + n2);
  float* prec = rec + (size_t)ne * T;
  float* env = prec + (size_t)ne * T;
  float* cconf = env + (size_t)ne * T;
  float* x1000 = cconf + nn;
  float* x101 = x1000 + AP_PTS;
  int* n_pred = reinterpret_cast<int*>(x101 + AP_COCO);
  int* n_lab = n_pred + max_classes;
  int* seg_start = n_lab + max_classes;
  int* prec_row = seg_start + max_classes;
  int* cnt = prec_row + max_classes;  // [0] n_uniq, [1] n_prec, [2] best
  unsigned char* ctp = reinterpret_cast<unsigned char*>(cnt + 4);
  int rc = YB_OK;
  auto fail = [&](int code) { cudaFreeAsync(scratch, s); return code; };
  std::vector<float> h1000, h101;
  linspace01(AP_PTS, h1000);
  linspace01(AP_COCO, h101);
  if (cudaMemcpyAsync(x1000, h1000.data(), AP_PTS * 4, cudaMemcpyHostToDevice, s) != cudaSuccess ||
      cudaMemcpyAsync(x101, h101.data(), AP_COCO * 4, cudaMemcpyHostToDevice, s) != cudaSuccess ||
      cudaStreamSynchronize(s) != cudaSuccess ||  // the two host vectors are temporaries
      cudaMemsetAsync(n_pred, 0, i_count * 4, s) != cudaSuccess ||
      cudaMemsetAsync(ap, 0, (size_t)max_classes * T * 4, s) != cudaSuccess ||
      cudaMemsetAsync(p_curve, 0, (size_t)max_classes * AP_PTS * 4, s) != cudaSuccess ||
      cudaMemsetAsync(r_curve, 0, (size_t)max_classes * AP_PTS * 4, s) != cudaSuccess ||
      cudaMemsetAsync(prec_values, 0, (size_t)max_classes * AP_PTS * 4, s) != cudaSuccess) {
    set_error(std::string("yb_ap_per_class: ") + cudaGetErrorString(cudaGetLastError()));
    return fail(YB_ERR_CUDA);
  }
  if (m > 0) target_hist_kernel<<<(m + 255) / 256, 256, 0, s>>>(target_cls, m, max_classes, n_lab);
  if (n > 0) {
    conf_keys_kernel<<<(n2 + 255) / 256, 256, 0, s>>>(conf, n, n2, k1);
    if ((rc = sort_keys(k1, n2, s))) return fail(rc);
    class_keys_kernel<<<(n2 + 255) / 256, 256, 0, s>>>(k1, pred_cls, n, n2, max_classes, k2, n_pred);
    if ((rc = sort_keys(k2, n2, s))) return fail(rc);
    gather_kernel<<<(n + 255) / 256, 256, 0, s>>>(k1, k2, conf, tp, n, T, cconf, ctp);
  }
  classes_kernel<<<1, 1024, 0, s>>>(n_pred, n_lab, max_classes, seg_start, unique_classes, cnt);
  prec_rows_kernel<<<1, 32, 0, s>>>(unique_classes, cnt, n_pred, n_lab, prec_row, cnt + 1);
  if (n > 0) {
    pr_kernel<<<dim3(max_classes, T), 1024, 0, s>>>(unique_classes, cnt, seg_start, n_pred, n_lab, ctp, n, ne, rec, prec, env);
    ap_kernel<<<dim3(max_classes, T), 128, 0, s>>>(unique_classes, cnt, seg_start, n_pred, n_lab, rec, env, ne, T, x101, ap);
    curves_kernel<<<max_classes, 1024, 0, s>>>(unique_classes, cnt, seg_start, n_pred, n_lab, cconf, rec, prec, env, ne, x1000, p_curve, r_curve,
                                               prec_values, prec_row);
  }
  f1_kernel<<<1, 1024, 0, s>>>(unique_classes, cnt, n_lab, p_curve, r_curve, f1_curve, 1e-16f, p, r, f1, tp_out, fp_out, cnt + 2);
  cudaError_t ce = cudaGetLastError();
  if (ce == cudaSuccess) ce = cudaMemcpyAsync(counts_host, cnt, 3 * sizeof(int), cudaMemcpyDeviceToHost, s);
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(s);
  cudaFreeAsync(scratch, s);
  if (ce != cudaSuccess) { set_error(std::string("yb_ap_per_class: ") + cudaGetErrorString(ce)); return YB_ERR_CUDA; }
  return YB_OK;
}

}  // extern "C"
