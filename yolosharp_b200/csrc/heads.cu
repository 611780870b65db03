// Decode tails of the other Detect-family heads and the rotated NMS (SURVEY.md section 8(f) row f4).
//
//   yb_obb_decode    `Obb.decode_bboxes` = `Tal.dist2rbox(dfl(boxes), angle, anchors, dim: 1) * strides` with
//                    angle = (sigmoid(raw) - 0.25) * pi  (Modules/Head.cs:423-436, Utils/Tal.cs:389-408, DFL Block.cs:15-45)
//                    + class sigmoid, written as the reference's (B, 4 + nc + 1, A) inference tensor (Head.cs:410-416)
//   yb_pose_decode   `Pose.kpts_decode` (Modules/Head.cs:595-609): x, y -> (v * 2 + anchor - 0.5) * stride, visibility ->
//                    sigmoid when keypoint_dim == 3
//   yb_probiou       `Metrics.batch_probiou` (Utils/Metrics.cs:223-254, covariance Metrics.cs:260-280)
//   yb_nms_rotated   `Ops.nms_rotated(boxes, scores, threshold)` with use_triu (Utils/Ops.cs:373-401): sort by score,
//                    keep box j iff no HIGHER-scored box i has probiou(i, j) >= threshold (a matrix test, not the greedy
//                    pass of the axis-aligned NMS), return the kept original indices in score order
// fp32 throughout; sin / cos / exp / log are the CUDA library functions (the oracle runs libm through torch on the CPU:
// results agree to a few ulps, tests use 1e-5 and keep IoUs away from the threshold).
#include <algorithm>
#include <string>

#include "common.cuh"

namespace yb {

__global__ void obb_decode_kernel(const float* __restrict__ box, const float* __restrict__ cls, const float* __restrict__ ang,
                                  const float* __restrict__ anchors, const float* __restrict__ strides, int B, int A, int nc,
                                  int reg_max, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * A) return;
  const int b = (int)(i / A), a = (int)(i - (long long)b * A);
  float d[4];
  for (int sd = 0; sd < 4; sd++) {  // DFL: softmax over reg_max bins, expectation with weights 0 .. reg_max-1
    const float* p = box + ((size_t)b * 4 * reg_max + (size_t)sd * reg_max) * A + a;
    float mx = -INFINITY;
    for (int j = 0; j < reg_max; j++) mx = fmaxf(mx, p[(size_t)j * A]);
    float sum = 0.f, ex = 0.f;
    for (int j = 0; j < reg_max; j++) {
      const float e = expf(p[(size_t)j * A] - mx);
      sum += e;
      ex += e * (float)j;
    }
    d[sd] = ex / sum;
  }
  const float angle = (1.0f / (1.0f + expf(-ang[(size_t)b * A + a])) - 0.25f) * 3.14159265358979323846f;
  const float c = cosf(angle), s = sinf(angle);
  const float xf = (d[2] - d[0]) * 0.5f, yf = (d[3] - d[1]) * 0.5f;  // ((rb - lt) / 2)
  const float st = strides[a];
  const size_t C = 4 + nc + 1;
  float* o = out + (size_t)b * C * A + a;
  o[0] = (xf * c - yf * s + anchors[a]) * st;
  o[(size_t)A] = (xf * s + yf * c + anchors[(size_t)A + a]) * st;
  o[(size_t)2 * A] = (d[0] + d[2]) * st;
  o[(size_t)3 * A] = (d[1] + d[3]) * st;
  for (int k = 0; k < nc; k++) o[(size_t)(4 + k) * A] = 1.0f / (1.0f + expf(-cls[((size_t)b * nc + k) * A + a]));
  o[(size_t)(4 + nc) * A] = angle;
}

__global__ void pose_decode_kernel(const float* __restrict__ kpts, const float* __restrict__ anchors,
                                   const float* __restrict__ strides, int B, int A, int nk, int ndim, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * nk * A) return;
  const int a = (int)(i % A);
  const int ch = (int)((i / A) % nk);
  const int comp = ch % ndim;
  const float v = kpts[i];
  float r;
  if (comp == 0) r = (v * 2.0f + (anchors[a] - 0.5f)) * strides[a];
  else if (comp == 1) r = (v * 2.0f + (anchors[(size_t)A + a] - 0.5f)) * strides[a];
  else r = 1.0f / (1.0f + expf(-v));
  out[i] = r;
}

// covariance of a rotated box (x, y, w, h, r): a = w^2/12, b = h^2/12 rotated by r (Metrics.cs:260-280)
__device__ __forceinline__ void obb_cov(const float* o, float& a, float& b, float& c) {
  const float ga = o[2] * o[2] / 12.0f, gb = o[3] * o[3] / 12.0f;
  const float cs = cosf(o[4]), sn = sinf(o[4]);
  const float c2 = cs * cs, s2 = sn * sn;
  a = ga * c2 + gb * s2;
  b = ga * s2 + gb * c2;
  c = (ga - gb) * cs * sn;
}
__device__ __forceinline__ float probiou_dev(const float* o1, const float* o2, float eps) {
  float a1, b1, c1, a2, b2, c2;
  obb_cov(o1, a1, b1, c1);
  obb_cov(o2, a2, b2, c2);
  const float x1 = o1[0], y1 = o1[1], x2 = o2[0], y2 = o2[1];
  const float sa = a1 + a2, sb = b1 + b2, sc = c1 + c2;
  const float den = sa * sb - sc * sc + eps;
  const float t1 = ((sa * (y1 - y2) * (y1 - y2) + sb * (x1 - x2) * (x1 - x2)) / den) * 0.25f;
  const float t2 = ((sc * (x2 - x1) * (y1 - y2)) / den) * 0.5f;
  const float d1 = fmaxf(a1 * b1 - c1 * c1, 0.f), d2 = fmaxf(a2 * b2 - c2 * c2, 0.f);
  const float t3 = logf((sa * sb - sc * sc) / (4.0f * sqrtf(d1 * d2) + eps) + eps) * 0.5f;
  const float bd = fminf(fmaxf(t1 + t2 + t3, eps), 100.0f);
  const float hd = sqrtf(1.0f - expf(-bd) + eps);
  return 1.0f - hd;
}

__global__ void probiou_kernel(const float* __restrict__ o1, int n, const float* __restrict__ o2, int m, float eps,
                               float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)n * m) return;
  const int r = (int)(i / m), c = (int)(i - (long long)r * m);
  out[i] = probiou_dev(o1 + (size_t)r * 5, o2 + (size_t)c * 5, eps);
}

// ---- rotated NMS ----
// keys: (~orderable(score) << 32) | index, ascending = score-descending, equal scores by index (torch.argsort leaves
// ties unspecified)
__global__ void rnms_keys_kernel(const float* __restrict__ scores, int n, int P2, unsigned long long* __restrict__ keys) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P2) return;
  if (i < n) {
    const unsigned u = __float_as_uint(scores[i]);
    const unsigned k = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    keys[i] = ((unsigned long long)(~k) << 32) | (unsigned)i;
  } else {
    keys[i] = ~0ull;
  }
}
__global__ void rnms_bitonic_step(unsigned long long* __restrict__ keys, int P2, int k, int j) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P2) return;
  const int ixj = i ^ j;
  if (ixj > i) {
    const unsigned long long x = keys[i], y = keys[ixj];
    if ((x > y) == ((i & k) == 0)) { keys[i] = y; keys[ixj] = x; }
  }
}
// box (sorted position j) survives iff no earlier sorted box overlaps it with probiou >= thr
__global__ void rnms_suppress_kernel(const float* __restrict__ boxes, const unsigned long long* __restrict__ keys, int n, float thr,
                                     unsigned char* __restrict__ alive) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const float* bj = boxes + (size_t)(unsigned)(keys[j] & 0xffffffffu) * 5;
  const float mine[5] = {bj[0], bj[1], bj[2], bj[3], bj[4]};
  unsigned char ok = 1;
  for (int i = 0; i < j; i++) {
    const float* bi = boxes + (size_t)(unsigned)(keys[i] & 0xffffffffu) * 5;
    if (probiou_dev(bi, mine, 1e-7f) >= thr) { ok = 0; break; }
  }
  alive[j] = ok;
}
__global__ void rnms_compact_kernel(const unsigned long long* __restrict__ keys, const unsigned char* __restrict__ alive, int n,
                                    int* __restrict__ keep, int* __restrict__ count) {
  __shared__ int wsum[32];
  __shared__ int run;
  if (threadIdx.x == 0) run = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int base = 0; base < n; base += 1024) {
    const int j = base + threadIdx.x;
    const bool f = j < n && alive[j];
    const unsigned m = __ballot_sync(0xffffffffu, f);
    if (lane == 0) wsum[warp] = __popc(m);
    __syncthreads();
    int off = run;
    for (int w = 0; w < warp; w++) off += wsum[w];
    if (f) keep[off + __popc(m & ((1u << lane) - 1u))] = (int)(unsigned)(keys[j] & 0xffffffffu);
    __syncthreads();
    if (threadIdx.x == 0) {
      int t = 0;
      for (int w = 0; w < 32; w++) t += wsum[w];
      run += t;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) *count = run;
}

}  // namespace yb

using namespace yb;

extern "C" {

int32_t yb_obb_decode(const float* box_logits, const float* cls_logits, const float* angle_logits, const float* anchors,
                      const float* strides, int32_t batch, int32_t anchors_n, int32_t nc, int32_t reg_max, float* out, void* stream) {
  if (!box_logits || !cls_logits || !angle_logits || !anchors || !strides || !out || batch <= 0 || anchors_n <= 0 || nc <= 0 || reg_max <= 0) {
    set_error("yb_obb_decode: bad argument");
    return YB_ERR_INVALID_ARG;
  }
  if (!have_device("yb_obb_decode")) return YB_ERR_NO_DEVICE;
  const long long n = (long long)batch * anchors_n;
  obb_decode_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(box_logits, cls_logits, angle_logits, anchors, strides,
                                                                                    batch, anchors_n, nc, reg_max, out);
  YB_CUDA_CHECK(cudaGetLastError());
  return YB_OK;
}

int32_t yb_pose_decode(const float* kpts, const float* anchors, const float* strides, int32_t batch, int32_t anchors_n, int32_t nk,
                       int32_t keypoint_dim, float* out, void* stream) {
  if (!kpts || !anchors || !strides || !out || batch <= 0 || anchors_n <= 0 || nk <= 0 || (keypoint_dim != 2 && keypoint_dim != 3) ||
      nk % keypoint_dim) {
    set_error("yb_pose_decode: bad argument (keypoint_dim must be 2 or 3 and divide the channel count)");
    return YB_ERR_INVALID_ARG;
  }
  if (!have_device("yb_pose_decode")) return YB_ERR_NO_DEVICE;
  const long long n = (long long)batch * nk * anchors_n;
  pose_decode_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(kpts, anchors, strides, batch, anchors_n, nk,
                                                                                     keypoint_dim, out);
  YB_CUDA_CHECK(cudaGetLastError());
  return YB_OK;
}

int32_t yb_probiou(const float* obb1, int32_t n, const float* obb2, int32_t m, float eps, float* out, void* stream) {
  if (!obb1 || !obb2 || !out || n < 0 || m < 0) { set_error("yb_probiou: bad argument"); return YB_ERR_INVALID_ARG; }
  if (!have_device("yb_probiou")) return YB_ERR_NO_DEVICE;
  const long long t = (long long)n * m;
  if (t == 0) return YB_OK;
  probiou_kernel<<<(unsigned)((t + 255) / 256), 256, 0, (cudaStream_t)stream>>>(obb1, n, obb2, m, eps, out);
  YB_CUDA_CHECK(cudaGetLastError());
  return YB_OK;
}

int32_t yb_nms_rotated(const float* boxes, const float* scores, int32_t n, float threshold, int32_t* keep, int32_t* count,
                       void* stream) {
  if (!keep || !count || n < 0 || (n > 0 && (!boxes || !scores))) { set_error("yb_nms_rotated: bad argument"); return YB_ERR_INVALID_ARG; }
  if (!have_device("yb_nms_rotated")) return YB_ERR_NO_DEVICE;
  cudaStream_t s = (cudaStream_t)stream;
  if (n == 0) {
    YB_CUDA_CHECK(cudaMemsetAsync(count, 0, sizeof(int32_t), s));
    return YB_OK;
  }
  int P2 = 1;
  while (P2 < n) P2 <<= 1;
  unsigned long long* keys = nullptr;
  unsigned char* alive = nullptr;
  YB_CUDA_CHECK(cudaMallocAsync((void**)&keys, (size_t)P2 * sizeof(unsigned long long), s));
  YB_CUDA_CHECK(cudaMallocAsync((void**)&alive, (size_t)n, s));
  const unsigned gb = (unsigned)((P2 + 255) / 256);
  rnms_keys_kernel<<<gb, 256, 0, s>>>(scores, n, P2, keys);
  for (int k = 2; k <= P2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) rnms_bitonic_step<<<gb, 256, 0, s>>>(keys, P2, k, j);
  rnms_suppress_kernel<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(boxes, keys, n, threshold, alive);
  rnms_compact_kernel<<<1, 1024, 0, s>>>(keys, alive, n, keep, count);
  cudaError_t ce = cudaGetLastError();
  cudaFreeAsync(keys, s);
  cudaFreeAsync(alive, s);
  YB_CUDA_CHECK(ce);
  return YB_OK;
}

}  // extern "C"
