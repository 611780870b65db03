// NMS-free ("end2end") post-processing of the Detect head on the GPU.
//
// Replaces `Detect.postprocess` + `Detect.get_topk_index` (Modules/Head.cs:117-127, 175-196), the tail the reference runs
// instead of non_max_suppression when the head is end2end (`Config.End2End` defaults to true, Data/Config.cs:239):
//     scores (B, A, nc)  ->  the k = min(max_det, A) anchors with the largest best-class score        (topk #1)
//                        ->  the k largest of the k x nc (anchor, class) scores of those anchors       (topk #2)
//                        ->  rows (x, y, w, h, score, class), sorted by score
// One CTA per image.  Both selections are radix selects on order-preserving integer keys of the fp32 scores (four
// 8-bit digit passes over a shared-memory histogram: exact k-th value, no sort of the 8 400 / 24 000 candidates),
// followed by an index-ordered compaction; only the final k rows are sorted (bitonic, shared memory).
// Ties: torch.topk leaves the choice among equal scores unspecified; here equal scores are taken in index order
// (anchor index for the first selection, anchor-major (anchor, class) order for the second, and rows of equal score
// are emitted in that order).
#include <algorithm>
#include <string>

#include "common.cuh"

namespace yb {

constexpr int TK_THREADS = 1024;
constexpr int TK_MAX_K = 1024;

__device__ __forceinline__ unsigned tk_key(float v) {
  const unsigned u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);  // ascending integer order == ascending float order
}

// k-th largest key of n values produced by `val(i)`: returns the key T and, through n_gt, how many keys are > T.
template <typename F>
__device__ unsigned tk_radix_select(F val, int n, int k, unsigned* hist, unsigned* bc, int* n_gt) {
  unsigned prefix = 0, mask = 0;
  int need = k, above = 0;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += TK_THREADS) hist[i] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += TK_THREADS) {
      const unsigned key = tk_key(val(i));
      if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int acc = 0, d = 255;
      for (; d > 0; d--) {
        if (acc + (int)hist[d] >= need) break;
        acc += (int)hist[d];
      }
      bc[0] = (unsigned)d;
      bc[1] = (unsigned)acc;
    }
    __syncthreads();
    const unsigned d = bc[0];
    above += (int)bc[1];
    need -= (int)bc[1];
    prefix |= d << shift;
    mask |= 255u << shift;
    __syncthreads();
  }
  *n_gt = above;
  return prefix;
}

// Index-ordered compaction of the elements with key > T plus the first `need_eq` elements with key == T.
// emit(slot, i) is called once per selected element, slot = its rank in index order.
template <typename F, typename E>
__device__ void tk_compact(F val, int n, unsigned T, int need_eq, unsigned* wsum, int* run, E emit) {
  if (threadIdx.x == 0) { run[0] = 0; run[1] = 0; }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int base = 0; base < n; base += TK_THREADS) {
    const int i = base + threadIdx.x;
    unsigned key = 0;
    bool gt = false, eq = false;
    if (i < n) {
      key = tk_key(val(i));
      gt = key > T;
      eq = key == T;
    }
    const unsigned mg = __ballot_sync(0xffffffffu, gt), me = __ballot_sync(0xffffffffu, eq);
    if (lane == 0) { wsum[warp] = __popc(mg); wsum[32 + warp] = __popc(me); }
    __syncthreads();
    int g0 = run[0], e0 = run[1];
    for (int w = 0; w < warp; w++) { g0 += (int)wsum[w]; e0 += (int)wsum[32 + w]; }
    const int my_g = g0 + __popc(mg & ((1u << lane) - 1u)), my_e = e0 + __popc(me & ((1u << lane) - 1u));
    // selected elements in index order: every gt element, and eq elements while their rank among equals < need_eq
    const bool sel = gt || (eq && my_e < need_eq);
    if (sel) emit(my_g + min(my_e, need_eq), i);
    __syncthreads();
    if (threadIdx.x == 0) {
      int tg = 0, te = 0;
      for (int w = 0; w < 32; w++) { tg += (int)wsum[w]; te += (int)wsum[32 + w]; }
      run[0] += tg;
      run[1] += te;
    }
    __syncthreads();
  }
}

// pred (B, C = 4 + nc [+ extra], A) channel-major fp32 (the tensor yb_forward writes); out (B, k, 6); idx (B, k) or null
__global__ void __launch_bounds__(TK_THREADS, 1)
topk_postprocess_kernel(const float* __restrict__ pred, int C, int A, int nc, int k, int agnostic, float* __restrict__ best,
                        int* __restrict__ best_cls, float* __restrict__ out, int* __restrict__ idx_out) {
  __shared__ unsigned hist[256];
  __shared__ unsigned bc[2];
  __shared__ unsigned wsum[64];
  __shared__ int run[2];
  __shared__ int sel_anchor[TK_MAX_K];
  __shared__ unsigned long long skey[TK_MAX_K];
  const int b = blockIdx.x;
  const float* P = pred + (size_t)b * C * A;
  float* m = best + (size_t)b * A;
  int* mc = best_cls + (size_t)b * A;
  // best class score per anchor (threads over anchors: coalesced rows of the channel-major tensor)
  for (int a = threadIdx.x; a < A; a += TK_THREADS) {
    float v = P[(size_t)4 * A + a];
    int c0 = 0;
    for (int c = 1; c < nc; c++) {
      const float s = P[(size_t)(4 + c) * A + a];
      if (s > v) { v = s; c0 = c; }
    }
    m[a] = v;
    mc[a] = c0;
  }
  __syncthreads();
  // ---- topk #1: k anchors by best-class score ----
  int n_gt;
  auto val1 = [&](int i) { return m[i]; };
  const unsigned T1 = tk_radix_select(val1, A, k, hist, bc, &n_gt);
  tk_compact(val1, A, T1, k - n_gt, wsum, run, [&](int slot, int i) { sel_anchor[slot] = i; });
  __syncthreads();
  int P2 = 1;
  while (P2 < k) P2 <<= 1;
  if (agnostic) {
    // (scores, labels) = scores.max(-1); topk over anchors; rows sorted by score
    for (int j = threadIdx.x; j < P2; j += TK_THREADS)
      skey[j] = j < k ? ((unsigned long long)(~tk_key(m[sel_anchor[j]])) << 32) | (unsigned)sel_anchor[j] : ~0ull;
  } else {
    // ---- topk #2: k of the k x nc (selected anchor, class) scores ----
    const int n2 = k * nc;
    auto val2 = [&](int f) { const int j = f / nc; return P[(size_t)(4 + f - j * nc) * A + sel_anchor[j]]; };
    int n_gt2;
    const unsigned T2 = tk_radix_select(val2, n2, k, hist, bc, &n_gt2);
    for (int j = threadIdx.x; j < P2; j += TK_THREADS) skey[j] = ~0ull;
    __syncthreads();
    tk_compact(val2, n2, T2, k - n_gt2, wsum, run,
               [&](int slot, int f) { skey[slot] = ((unsigned long long)(~tk_key(val2(f))) << 32) | (unsigned)f; });
  }
  __syncthreads();
  for (int kk = 2; kk <= P2; kk <<= 1)
    for (int j = kk >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < P2; i += TK_THREADS) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long x = skey[i], y = skey[ixj];
          if ((x > y) == ((i & kk) == 0)) { skey[i] = y; skey[ixj] = x; }
        }
      }
      __syncthreads();
    }
  for (int j = threadIdx.x; j < k; j += TK_THREADS) {
    const unsigned f = (unsigned)(skey[j] & 0xffffffffu);
    int a, cls;
    if (agnostic) { a = (int)f; cls = mc[a]; }
    else { const int jj = (int)f / nc; a = sel_anchor[jj]; cls = (int)f - jj * nc; }
    float* o = out + ((size_t)b * k + j) * 6;
    o[0] = P[a]; o[1] = P[(size_t)A + a]; o[2] = P[(size_t)2 * A + a]; o[3] = P[(size_t)3 * A + a];
    o[4] = P[(size_t)(4 + cls) * A + a];
    o[5] = (float)cls;
    if (idx_out) idx_out[(size_t)b * k + j] = a;
  }
}

int topk_postprocess_launch(const float* pred, int B, int C, int A, int nc, int max_det, int agnostic, float* out, int* idx_out,
                            cudaStream_t s) {
  const int k = std::min(max_det, A);
  if (k <= 0 || k > TK_MAX_K) { set_error("yb_topk_postprocess: max_det must be in [1, 1024]"); return YB_ERR_INVALID_ARG; }
  if (nc <= 0 || C < 4 + nc) { set_error("yb_topk_postprocess: channels < 4 + nc"); return YB_ERR_SHAPE; }
  float* best = nullptr;
  int* best_cls = nullptr;
  YB_CUDA_CHECK(cudaMallocAsync((void**)&best, (size_t)B * A * sizeof(float), s));
  YB_CUDA_CHECK(cudaMallocAsync((void**)&best_cls, (size_t)B * A * sizeof(int), s));
  topk_postprocess_kernel<<<B, TK_THREADS, 0, s>>>(pred, C, A, nc, k, agnostic, best, best_cls, out, idx_out);
  YB_CUDA_CHECK(cudaGetLastError());
  YB_CUDA_CHECK(cudaFreeAsync(best, s));
  YB_CUDA_CHECK(cudaFreeAsync(best_cls, s));
  return 0;
}

}  // namespace yb

using namespace yb;

extern "C" int32_t yb_topk_postprocess(const float* pred, int32_t batch, int32_t channels, int32_t anchors, int32_t nc,
                                       int32_t max_det, int32_t agnostic, float* out, int32_t* idx, void* stream) {
  if (!pred || !out || batch <= 0 || anchors <= 0) { set_error("yb_topk_postprocess: bad argument"); return YB_ERR_INVALID_ARG; }
  if (!have_device("yb_topk_postprocess")) return YB_ERR_NO_DEVICE;
  return topk_postprocess_launch(pred, batch, channels, anchors, nc, max_det, agnostic, out, idx, (cudaStream_t)stream);
}
