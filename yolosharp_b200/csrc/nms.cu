// GPU non-max suppression + mask post-processing.
//
// Restates Utils/Ops.cs:239-371 (`non_max_suppression`, non-rotated / non-end2end path) of the
// reference, including the torchvision.ops.nms core it calls at :357, with bit-identical
// arithmetic: every fp32 op below is an explicit round-to-nearest intrinsic so nvcc cannot
// contract mul+add into FMA (the CPU kernel is compiled without FMA contraction).
//
//  per image (one CTA, 1024 threads):
//   1. candidate scan  : conf = max_c prob[c][a], j = first argmax; keep conf > conf_thres
//                        (Ops.cs:272, 325-328).  64-bit key = (~bits(conf) << 32) | anchor << 12 | j
//   2. bitonic sort    : ascending key == score descending, anchor index ascending on ties
//                        (torchvision sorts scores with a stable descending sort); truncate to
//                        max_nms (Ops.cs:338-342)
//   3. greedy suppress : boxes offset by cls*max_wh in fp32 (Ops.cs:345,356).
//        fast path (<= 4096 candidates, every box inside (-0.49, 0.49) * max_wh): the class offsets then
//          make boxes of different classes disjoint, so IoU across classes is exactly 0 and the greedy
//          pass decomposes into independent per-class passes.  Candidates are re-sorted class-major
//          (score order inside a class), each warp runs whole class segments 32 candidates at a time
//          (kept list of the class, then a ballot-driven resolve inside the chunk), and the kept flags are
//          compacted in score order - the same set in the same order as the sequential pass.
//        general path: candidates are consumed in chunks of 32 by the whole CTA: a 32x32 IoU bit-matrix
//          inside the chunk plus a check against the kept list, then a 32-step serial resolve.  Stops at
//          max_det kept boxes (Ops.cs:360 - later boxes cannot change earlier ones).
#include <cstdlib>

#include "common.cuh"

namespace yb {

constexpr int NMS_THREADS = 1024;
constexpr int NMS_SMEM_KEYS = 16384;  // candidates sortable in shared memory (128 KB of keys)
constexpr int NMS_FAST_N = 4096;      // candidates the class-wise fast path handles
constexpr int NMS_LONG_SEG = 128;     // longer class segments are processed by the whole CTA
constexpr int NMS_MAX_DET_CAP = 1024;
constexpr int NMS_SC = 1024;  // sorted candidates gathered into shared memory per super-chunk

struct Box5 {
  float x1, y1, x2, y2, area;
};
// shared memory: [64-bit keys of NMS_SMEM_KEYS candidates][union of the two greedy paths]
//   general path: kept[1024] + super-chunk boxes/rows/anchors + rowmask
//   fast path   : float4 boxes + 32-bit class-major keys + keep flags + segment starts, NMS_FAST_N each
constexpr size_t NMS_KEYS_SMEM = (size_t)NMS_SMEM_KEYS * 8;
constexpr size_t NMS_GENERAL_SMEM = (NMS_MAX_DET_CAP + NMS_SC) * sizeof(Box5) + NMS_SC * 6 * 4 + NMS_SC * 4 + 32 * 4;
constexpr size_t NMS_FAST_SMEM = (size_t)NMS_FAST_N * (16 + 4 + 1 + 2) + 64 * 4;
constexpr size_t NMS_TOTAL_SMEM =
    NMS_KEYS_SMEM + (NMS_GENERAL_SMEM > NMS_FAST_SMEM ? NMS_GENERAL_SMEM : NMS_FAST_SMEM) + 64;


// IoU > thr test with the exact op order of torchvision's CPU kernel (nms_kernel_impl):
//   w = max(0, xx2-xx1); h = max(0, yy2-yy1); inter = w*h; ovr = inter / (iarea + area_j - inter)
__device__ __forceinline__ bool iou_gt(const Box5& a, const Box5& b, float thr) {
  const float xx1 = fmaxf(a.x1, b.x1), yy1 = fmaxf(a.y1, b.y1);
  const float xx2 = fminf(a.x2, b.x2), yy2 = fminf(a.y2, b.y2);
  const float w = fmaxf(0.0f, __fsub_rn(xx2, xx1));
  const float h = fmaxf(0.0f, __fsub_rn(yy2, yy1));
  // disjoint boxes (the common case): inter = 0 -> ovr = 0 or NaN, never > thr (thr >= 0); skip the IEEE division
  if (!(w > 0.0f && h > 0.0f)) return false;
  const float inter = __fmul_rn(w, h);
  const float ovr = __fdiv_rn(inter, __fsub_rn(__fadd_rn(a.area, b.area), inter));
  return ovr > thr;  // NaN (0/0) compares false, as on the CPU
}

__device__ __forceinline__ bool iou_gt4(const float4& a, const float4& b, float thr) {
  Box5 x, y;
  x.x1 = a.x; x.y1 = a.y; x.x2 = a.z; x.y2 = a.w;
  x.area = __fmul_rn(__fsub_rn(a.z, a.x), __fsub_rn(a.w, a.y));
  y.x1 = b.x; y.y1 = b.y; y.x2 = b.z; y.y2 = b.w;
  y.area = __fmul_rn(__fsub_rn(b.z, b.x), __fsub_rn(b.w, b.y));
  return iou_gt(x, y, thr);
}

// Stage 1 (all SMs): per anchor best class + confidence (Ops.cs:272, 325-328).  conf = -1 marks
// "not a candidate"; strict '>' keeps the FIRST maximal class like torch.max.
__global__ void __launch_bounds__(256) nms_scan_kernel(const float* __restrict__ pred, int C, int A, int nc,
                                                       float conf_thres, float* __restrict__ sconf,
                                                       int* __restrict__ scls) {
  const int b = blockIdx.y;
  const int a = blockIdx.x * 256 + threadIdx.x;
  if (a >= A) return;
  const float* P = pred + (size_t)b * C * A + (size_t)4 * A + a;
  float best = P[0];
  int bj = 0;
  int c = 1;
  for (; c + 8 <= nc; c += 8) {  // 8 independent loads in flight per thread
    float v[8];
#pragma unroll
    for (int u = 0; u < 8; u++) v[u] = P[(size_t)(c + u) * A];
#pragma unroll
    for (int u = 0; u < 8; u++)
      if (v[u] > best) { best = v[u]; bj = c + u; }
  }
  for (; c < nc; c++) {
    const float v = P[(size_t)c * A];
    if (v > best) { best = v; bj = c; }
  }
  sconf[(size_t)b * A + a] = best > conf_thres ? best : -1.0f;
  scls[(size_t)b * A + a] = bj;
}

__global__ void __launch_bounds__(NMS_THREADS, 1)
nms_kernel(const float* __restrict__ pred, int C, int A, int nc, float conf_thres, float iou_thres,
           int max_det, int max_nms, float max_wh, float* __restrict__ dets, int* __restrict__ counts,
           int* __restrict__ keep_idx, unsigned long long* __restrict__ gkeys, int key_cap,
           const float* __restrict__ sconf, const int* __restrict__ scls, int fast_n) {
  extern __shared__ __align__(16) unsigned char nms_smem[];
  const int b = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* P = pred + (size_t)b * C * A;
  const int extra = C - 4 - nc;
  const int row_w = 6 + extra;

  // shared carve-up
  unsigned* misc = reinterpret_cast<unsigned*>(nms_smem);                // [8]: n_cand, supp, n_seg, kept_n, ...
  unsigned long long* skeys = reinterpret_cast<unsigned long long*>(nms_smem + 64);
  unsigned char* un = nms_smem + 64 + NMS_KEYS_SMEM;
  // general path
  Box5* kept = reinterpret_cast<Box5*>(un);                              // [NMS_MAX_DET_CAP]
  Box5* cbox = kept + NMS_MAX_DET_CAP;                                   // [NMS_SC] super-chunk boxes (class-offset)
  float* craw = reinterpret_cast<float*>(cbox + NMS_SC);                 // [NMS_SC][6] raw rows
  int* canchor = reinterpret_cast<int*>(craw + NMS_SC * 6);              // [NMS_SC]
  unsigned* rowmask = reinterpret_cast<unsigned*>(canchor + NMS_SC);     // [32]
  // fast path
  float4* fbox = reinterpret_cast<float4*>(un);                          // [NMS_FAST_N] class-offset boxes by rank
  unsigned* ckey = reinterpret_cast<unsigned*>(fbox + NMS_FAST_N);       // [NMS_FAST_N] class << 12 | rank
  unsigned* frow = ckey + NMS_FAST_N;                                    // [32] chunk bit-matrix rows, [32..63] long segments
  unsigned short* segs = reinterpret_cast<unsigned short*>(frow + 64);   // [NMS_FAST_N] segment starts
  unsigned char* keepf = reinterpret_cast<unsigned char*>(segs + NMS_FAST_N);      // [NMS_FAST_N]
  // kept list of every class segment (ranks, at the segment's own positions).  It lives in the part of the key area
  // the fast path never touches (n <= NMS_FAST_N keys in use), so `ckey` is read-only while segments are processed:
  // a warp that scans past the end of its own segment reads a neighbour's class bits, never data being written.
  unsigned short* klist = reinterpret_cast<unsigned short*>(skeys + NMS_FAST_N);   // [NMS_FAST_N]
  unsigned long long* keys = gkeys + (size_t)b * key_cap;
  if (tid < 8) misc[tid] = 0;
  __syncthreads();

  // ---- 1. candidate compaction (per-anchor conf/class come from nms_scan_kernel) ----
  for (int a = tid; a < A; a += NMS_THREADS) {
    const float best = sconf[(size_t)b * A + a];
    if (best >= 0.0f) {
      const int bj = scls[(size_t)b * A + a];
      const unsigned slot = atomicAdd(&misc[0], 1u);
      if (slot < (unsigned)key_cap)
        keys[slot] = ((unsigned long long)(~__float_as_uint(best)) << 32) |
                     ((unsigned long long)(unsigned)a << 12) | (unsigned)bj;
    }
  }
  __syncthreads();
  int n = min((int)misc[0], key_cap);
  if (n == 0) {
    if (tid == 0) counts[b] = 0;
    return;
  }
  const bool in_smem = n <= NMS_SMEM_KEYS;
  if (in_smem) {  // sort in shared memory
    for (int i = tid; i < n; i += NMS_THREADS) skeys[i] = keys[i];
    keys = skeys;
    __syncthreads();
  }

  // ---- 2. bitonic sort (ascending) over the next power of two ----
  int P2 = 1;
  while (P2 < n) P2 <<= 1;
  for (int i = n + tid; i < P2; i += NMS_THREADS) keys[i] = ~0ull;
  __syncthreads();
  for (int k = 2; k <= P2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < P2; i += NMS_THREADS) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long x = keys[i], y = keys[ixj];
          const bool up = (i & k) == 0;
          if ((x > y) == up) { keys[i] = y; keys[ixj] = x; }
        }
      }
      __syncthreads();
    }
  }
  n = min(n, max_nms);

  // ---- 3a. class-wise fast path ----
  if (n <= fast_n) {
    const float lim = __fmul_rn(0.49f, max_wh);
    int bad = 0;
    for (int r = tid; r < n; r += NMS_THREADS) {
      const unsigned long long key = keys[r];
      const int a = (int)((key >> 12) & 0xFFFFF);
      const int j = (int)(key & 0xFFF);
      const float cx = P[a], cy = P[(size_t)A + a], w = P[(size_t)2 * A + a], h = P[(size_t)3 * A + a];
      const float hw = __fmul_rn(w, 0.5f), hh = __fmul_rn(h, 0.5f);
      const float x1 = __fsub_rn(cx, hw), y1 = __fsub_rn(cy, hh);
      const float x2 = __fadd_rn(cx, hw), y2 = __fadd_rn(cy, hh);
      const float off = __fmul_rn((float)j, max_wh);  // Ops.cs:345
      fbox[r] = make_float4(__fadd_rn(x1, off), __fadd_rn(y1, off), __fadd_rn(x2, off), __fadd_rn(y2, off));
      ckey[r] = ((unsigned)j << 12) | (unsigned)r;
      keepf[r] = 0;
      // x extents strictly inside (-0.49, 0.49) * max_wh => boxes of different classes cannot intersect
      if (!(fabsf(x1) < lim && fabsf(x2) < lim)) bad = 1;
    }
    bad = __syncthreads_or(bad);
    if (!bad) {
      int P2c = 1;
      while (P2c < n) P2c <<= 1;
      for (int i = n + tid; i < P2c; i += NMS_THREADS) ckey[i] = 0xFFFFFFFFu;
      __syncthreads();
      for (int k = 2; k <= P2c; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
          for (int i = tid; i < P2c; i += NMS_THREADS) {
            const int ixj = i ^ j;
            if (ixj > i) {
              const unsigned x = ckey[i], y = ckey[ixj];
              const bool up = (i & k) == 0;
              if ((x > y) == up) { ckey[i] = y; ckey[ixj] = x; }
            }
          }
          __syncthreads();
        }
      }
      // segment (= class) starts, in any order
      for (int i = tid; i < n; i += NMS_THREADS)
        if (i == 0 || (ckey[i] >> 12) != (ckey[i - 1] >> 12)) segs[atomicAdd(&misc[2], 1u)] = (unsigned short)i;
      __syncthreads();
      const int nseg = (int)misc[2];
      // short segments: one warp each
      for (int sg = warp; sg < nseg; sg += NMS_THREADS / 32) {
        const int s_begin = segs[sg];
        const unsigned cls = ckey[s_begin] >> 12;
        if (s_begin + NMS_LONG_SEG < n && (ckey[s_begin + NMS_LONG_SEG] >> 12) == cls) {  // long: whole CTA, below
          if (lane == 0) frow[32 + atomicAdd(&misc[4], 1u)] = (unsigned)s_begin;
          continue;
        }
        int kcount = 0;  // kept of this class so far; their keys are stored in place at ckey[s_begin ..]
        for (int s0 = s_begin; s0 < n && kcount < max_det; s0 += 32) {
          const unsigned ck = (s0 + lane < n) ? ckey[s0 + lane] : 0xFFFFFFFFu;
          const bool valid = (ck >> 12) == cls;
          const unsigned vmask = __ballot_sync(0xffffffffu, valid);
          if (!vmask) break;
          const int rank = (int)(ck & 0xFFF);
          const float4 mine = valid ? fbox[rank] : make_float4(0.f, 0.f, 0.f, 0.f);
          bool sup = false;
          for (int t = 0; t < kcount; t += 2) {  // two kept boxes per step (independent chains)
            const bool has1 = t + 1 < kcount;
            const float4 k0 = fbox[klist[s_begin + t]];
            const float4 k1 = fbox[klist[s_begin + (has1 ? t + 1 : t)]];
            const bool s0 = iou_gt4(k0, mine, iou_thres), s1 = iou_gt4(k1, mine, iou_thres);
            sup = sup || s0 || (has1 && s1);
          }
          unsigned alive = __ballot_sync(0xffffffffu, valid && !sup);
          unsigned keptmask = 0;
          while (alive) {
            const int i = __ffs(alive) - 1;
            keptmask |= 1u << i;
            float4 bi;
            bi.x = __shfl_sync(0xffffffffu, mine.x, i); bi.y = __shfl_sync(0xffffffffu, mine.y, i);
            bi.z = __shfl_sync(0xffffffffu, mine.z, i); bi.w = __shfl_sync(0xffffffffu, mine.w, i);
            const bool s2 = lane > i && iou_gt4(bi, mine, iou_thres);
            alive &= ~__ballot_sync(0xffffffffu, s2);
            alive &= ~(1u << i);
          }
          __syncwarp();
          if ((keptmask >> lane) & 1u) {
            klist[s_begin + kcount + __popc(keptmask & ((1u << lane) - 1u))] = (unsigned short)rank;
            keepf[rank] = 1;
          }
          __syncwarp();
          kcount += __popc(keptmask);
          if (vmask != 0xffffffffu) break;  // the segment ended inside this chunk
        }
      }
      __syncthreads();
      // long segments (> NMS_LONG_SEG candidates of one class; at most 31 of them): the whole CTA works on one
      // chunk of 32 at a time - warp g builds row g of the chunk's IoU bit-matrix and tests the chunk against
      // kept entries g, g+32, ...; warp 0 then resolves the chunk serially.  All operands are already in smem.
      const int nlong = (int)misc[4];
      for (int lg = 0; lg < nlong; lg++) {
        const int s_begin = (int)frow[32 + lg];
        const unsigned cls = ckey[s_begin] >> 12;
        int kcount = 0;
        for (int s0 = s_begin; s0 < n && kcount < max_det; s0 += 32) {
          const unsigned ck = (s0 + lane < n) ? ckey[s0 + lane] : 0xFFFFFFFFu;
          const bool valid = (ck >> 12) == cls;
          const unsigned vmask = __ballot_sync(0xffffffffu, valid);  // identical in every warp
          if (!vmask) break;
          const int rank = (int)(ck & 0xFFF);
          const float4 mine = valid ? fbox[rank] : make_float4(0.f, 0.f, 0.f, 0.f);
          {
            const unsigned ckr = (s0 + warp < n) ? ckey[s0 + warp] : 0xFFFFFFFFu;
            const bool rvalid = (ckr >> 12) == cls;
            const float4 rowb = rvalid ? fbox[ckr & 0xFFFu] : make_float4(0.f, 0.f, 0.f, 0.f);
            const bool hit = rvalid && valid && lane > warp && iou_gt4(rowb, mine, iou_thres);
            const unsigned m = __ballot_sync(0xffffffffu, hit);
            if (lane == 0) frow[warp] = m;
            bool sup = false;
            if (valid) {
              // two kept boxes per step: independent smem chains and IoU arithmetic in flight
              for (int k = warp; k < kcount; k += 64) {
                const float4 k0 = fbox[klist[s_begin + k]];
                const bool has1 = k + 32 < kcount;
                const float4 k1 = fbox[klist[s_begin + (has1 ? k + 32 : k)]];
                const bool s0 = iou_gt4(k0, mine, iou_thres), s1 = iou_gt4(k1, mine, iou_thres);
                sup = sup || s0 || (has1 && s1);
              }
            }
            const unsigned sm = __ballot_sync(0xffffffffu, sup);
            if (lane == 0 && sm) atomicOr(&misc[1], sm);
          }
          __syncthreads();
          if (warp == 0) {
            // serial resolve, one step per KEPT candidate: the lowest surviving index is kept and removes its row
            unsigned alive = ~(misc[1] | ~vmask);
            unsigned keptmask = 0;
            int kn = kcount;
            while (alive && kn < max_det) {
              const int i = __ffs(alive) - 1;
              keptmask |= 1u << i;
              alive &= ~(frow[i] | (1u << i));
              kn++;
            }
            if ((keptmask >> lane) & 1u) {
              klist[s_begin + kcount + __popc(keptmask & ((1u << lane) - 1u))] = (unsigned short)rank;
              keepf[rank] = 1;
            }
            __syncwarp();
            if (lane == 0) { misc[5] = (unsigned)kn; misc[1] = 0; }
          }
          __syncthreads();
          kcount = (int)misc[5];
          if (vmask != 0xffffffffu) break;
        }
        __syncthreads();
      }
      // ordered compaction of the kept flags (score order), 4 consecutive ranks per thread
      __shared__ unsigned s_wsum[32];
      const int r0 = tid * 4;
      int f[4], local = 0;
#pragma unroll
      for (int q = 0; q < 4; q++) { f[q] = (r0 + q < n) ? keepf[r0 + q] : 0; local += f[q]; }
      int incl = local;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += v;
      }
      if (lane == 31) s_wsum[warp] = (unsigned)incl;
      __syncthreads();
      if (warp == 0) {
        int v = (int)s_wsum[lane], inc2 = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const int u = __shfl_up_sync(0xffffffffu, inc2, d);
          if (lane >= d) inc2 += u;
        }
        s_wsum[lane] = (unsigned)(inc2 - v);  // exclusive warp offsets
        if (lane == 31) misc[3] = (unsigned)inc2;
      }
      __syncthreads();
      int pos = (int)s_wsum[warp] + incl - local;
#pragma unroll
      for (int q = 0; q < 4; q++) {
        if (f[q]) {
          if (pos < max_det) {
            const unsigned long long key = keys[r0 + q];
            const int a = (int)((key >> 12) & 0xFFFFF);
            const int j = (int)(key & 0xFFF);
            const float conf = __uint_as_float(~(unsigned)(key >> 32));
            const float cx = P[a], cy = P[(size_t)A + a], w = P[(size_t)2 * A + a], h = P[(size_t)3 * A + a];
            const float hw = __fmul_rn(w, 0.5f), hh = __fmul_rn(h, 0.5f);
            float* o = dets + ((size_t)b * max_det + pos) * row_w;
            o[0] = __fsub_rn(cx, hw); o[1] = __fsub_rn(cy, hh); o[2] = __fadd_rn(cx, hw); o[3] = __fadd_rn(cy, hh);
            o[4] = conf; o[5] = (float)j;
            for (int e = 0; e < extra; e++) o[6 + e] = P[(size_t)(4 + nc + e) * A + a];
            if (keep_idx) keep_idx[(size_t)b * max_det + pos] = a;
          }
          pos++;
        }
      }
      if (tid == 0) counts[b] = min((int)misc[3], max_det);
      return;
    }
    __syncthreads();  // fall through to the general path (its buffers overlay the fast-path arrays)
  }

  // ---- 3b. general greedy suppression: super-chunks of 1024 sorted candidates are gathered into shared
  //         memory by all threads (one global-latency exposure), then consumed 32 at a time ----
  int kept_n = 0;
  for (int sc0 = 0; sc0 < n && kept_n < max_det; sc0 += NMS_SC) {
    const int scn = min(NMS_SC, n - sc0);
    if (tid < scn) {
      const unsigned long long key = keys[sc0 + tid];
      const int a = (int)((key >> 12) & 0xFFFFF);
      const int j = (int)(key & 0xFFF);
      const float conf = __uint_as_float(~(unsigned)(key >> 32));
      const float cx = P[a], cy = P[(size_t)A + a], w = P[(size_t)2 * A + a], h = P[(size_t)3 * A + a];
      // xywh2xyxy (Ops.cs:76-79): x - w/2, x + w/2 (w/2 is exact)
      const float hw = __fmul_rn(w, 0.5f), hh = __fmul_rn(h, 0.5f);
      const float x1 = __fsub_rn(cx, hw), y1 = __fsub_rn(cy, hh);
      const float x2 = __fadd_rn(cx, hw), y2 = __fadd_rn(cy, hh);
      const float off = __fmul_rn((float)j, max_wh);  // Ops.cs:345
      Box5 bx;
      bx.x1 = __fadd_rn(x1, off); bx.y1 = __fadd_rn(y1, off);
      bx.x2 = __fadd_rn(x2, off); bx.y2 = __fadd_rn(y2, off);
      bx.area = __fmul_rn(__fsub_rn(bx.x2, bx.x1), __fsub_rn(bx.y2, bx.y1));
      cbox[tid] = bx;
      float* r = craw + tid * 6;
      r[0] = x1; r[1] = y1; r[2] = x2; r[3] = y2; r[4] = conf; r[5] = (float)j;
      canchor[tid] = a;
    }
    if (tid == 0) misc[1] = 0;
    __syncthreads();
    for (int s0 = 0; s0 < scn && kept_n < max_det; s0 += 32) {
      const int cnt = min(32, scn - s0);
      // phase A: warp g = row g of the intra-chunk IoU bit-matrix, then kept entries g, g+32, ...
      {
        const Box5 mine = cbox[s0 + min(lane, cnt - 1)];
        const Box5 rowb = cbox[s0 + min(warp, cnt - 1)];
        const bool hit = (warp < cnt) && (lane < cnt) && (lane > warp) && iou_gt(rowb, mine, iou_thres);
        const unsigned m = __ballot_sync(0xffffffffu, hit);
        if (lane == 0) rowmask[warp] = m;
        bool sup = false;
        if (lane < cnt)
          for (int k = warp; k < kept_n; k += 64) {  // two kept boxes per step (independent chains)
            const bool has1 = k + 32 < kept_n;
            const bool s0 = iou_gt(kept[k], mine, iou_thres), s1 = iou_gt(kept[has1 ? k + 32 : k], mine, iou_thres);
            sup = sup || s0 || (has1 && s1);
          }
        const unsigned sm = __ballot_sync(0xffffffffu, sup);
        if (lane == 0 && sm) atomicOr(&misc[1], sm);
      }
      __syncthreads();
      // phase B: serial resolve inside the chunk (warp 0, every lane runs the same bit loop)
      if (warp == 0) {
        unsigned alive = ~misc[1] & (cnt == 32 ? 0xffffffffu : ((1u << cnt) - 1u));
        unsigned keepmask = 0;
        int kn = kept_n;
        while (alive && kn < max_det) {  // one step per kept candidate
          const int i = __ffs(alive) - 1;
          keepmask |= 1u << i;
          alive &= ~(rowmask[i] | (1u << i));
          kn++;
        }
        if ((keepmask >> lane) & 1u) {
          const int pos = kept_n + __popc(keepmask & ((1u << lane) - 1u));
          kept[pos] = cbox[s0 + lane];
          float* o = dets + ((size_t)b * max_det + pos) * row_w;
          const float* r = craw + (s0 + lane) * 6;
#pragma unroll
          for (int q = 0; q < 6; q++) o[q] = r[q];
          const int a = canchor[s0 + lane];
          for (int q = 0; q < extra; q++) o[6 + q] = P[(size_t)(4 + nc + q) * A + a];
          if (keep_idx) keep_idx[(size_t)b * max_det + pos] = a;
        }
        __syncwarp();
        if (lane == 0) { misc[3] = (unsigned)kn; misc[1] = 0; }
      }
      __syncthreads();
      kept_n = (int)misc[3];
    }
    __syncthreads();  // the next super-chunk overwrites cbox/craw
  }
  if (tid == 0) counts[b] = kept_n;
}

int nms_launch(const float* pred, int B, int C, int A, int nc, float conf, float iou, int max_det,
               int max_nms, int max_wh, float* dets, int* counts, int* keep_idx, cudaStream_t s) {
  if (!(conf >= 0.f && conf <= 1.f)) {
    set_error("Invalid Confidence threshold " + std::to_string(conf) + ", valid values are between 0.0 and 1.0");
    return YB_ERR_INVALID_ARG;
  }
  if (!(iou >= 0.f && iou <= 1.f)) {
    set_error("Invalid IoU " + std::to_string(iou) + ", valid values are between 0.0 and 1.0");
    return YB_ERR_INVALID_ARG;
  }
  if (nc <= 0) nc = C - 4;
  if (B <= 0 || A <= 0 || C < 4 + nc || nc >= 4096 || A >= (1 << 20) || max_det <= 0 ||
      max_det > NMS_MAX_DET_CAP || max_nms <= 0) {
    set_error("yb_nms: unsupported shape (need nc < 4096, anchors < 2^20, 0 < max_det <= 1024)");
    return YB_ERR_SHAPE;
  }
  const int extra = C - 4 - nc;
  YB_CUDA_CHECK(cudaMemsetAsync(dets, 0, (size_t)B * max_det * (6 + extra) * sizeof(float), s));
  if (keep_idx) YB_CUDA_CHECK(cudaMemsetAsync(keep_idx, 0xFF, (size_t)B * max_det * sizeof(int), s));
  // candidate keys are compacted into global memory (every anchor may be a candidate); up to NMS_SMEM_KEYS of
  // them are then sorted in shared memory
  unsigned long long* gkeys = nullptr;
  int P2 = 1;
  while (P2 < A) P2 <<= 1;
  const int key_cap = P2;
  const size_t smem = NMS_TOTAL_SMEM;
  static bool pool_set = false;
  if (!pool_set) {
    // scratch comes from the stream-ordered pool on every call: keep freed blocks cached across host
    // synchronisation points (the default threshold 0 hands them back to the OS, and the next call pays for
    // mapping them again)
    int dev = 0;
    cudaMemPool_t pool = nullptr;
    unsigned long long keep_all = ~0ull;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess)
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep_all);
    cudaGetLastError();
    pool_set = true;
  }
  YB_CUDA_CHECK(cudaMallocAsync(&gkeys, (size_t)B * P2 * 8, s));
  YB_CUDA_CHECK(smem_limit((const void*)nms_kernel, smem, false));
  float* sconf = nullptr;
  YB_CUDA_CHECK(cudaMallocAsync(&sconf, (size_t)B * A * 8, s));  // conf[B][A] then cls[B][A]
  int* scls = reinterpret_cast<int*>(sconf + (size_t)B * A);
  static const int fast_n = getenv("YB_DEBUG_NMS_GENERAL") ? 0 : NMS_FAST_N;  // experiments only
  nms_scan_kernel<<<dim3((A + 255) / 256, B), 256, 0, s>>>(pred, C, A, nc, conf, sconf, scls);
  YB_CUDA_CHECK(cudaGetLastError());
  nms_kernel<<<B, NMS_THREADS, smem, s>>>(pred, C, A, nc, conf, iou, max_det, max_nms, (float)max_wh, dets, counts,
                                          keep_idx, gkeys, key_cap, sconf, scls, fast_n);
  YB_CUDA_CHECK(cudaGetLastError());
  YB_CUDA_CHECK(cudaFreeAsync(sconf, s));
  if (gkeys) YB_CUDA_CHECK(cudaFreeAsync(gkeys, s));
  return 0;
}

// ------------------------------------------------------------------------------------------
// Masks: Utils/Ops.cs:462-489 process_mask(upsample: true) with the CUDA branch of crop_mask
// (:437-447).  For every kept detection: m = coeff . proto (mh x mw), zero outside the box scaled
// to proto resolution (r >= x1 && r < x2 && c >= y1 && c < y2 in float), bilinear x(H/mh)
// upsample with align_corners=false (ATen upsample_bilinear2d), then > 0.
// One block per (detection, output row tile): the needed low-res rows are produced on the fly.
// ------------------------------------------------------------------------------------------
__global__ void masks_kernel(const float* __restrict__ proto, const float* __restrict__ dets,
                             const int* __restrict__ counts, int max_det, int mask_cap, int nm, int mh, int mw, int H, int W,
                             uint8_t* __restrict__ masks) {
  extern __shared__ float mk_smem[];  // [mh*mw] cropped low-res mask of this detection
  const int det = blockIdx.x, b = blockIdx.y;
  if (det >= counts[b]) return;  // grid.x = mask_cap: only the first mask_cap detections of an image get a mask
  const int row_w = 6 + nm;
  const float* d = dets + ((size_t)b * max_det + det) * row_w;
  const float* pr = proto + (size_t)b * nm * mh * mw;
  // width_ratio = (float)mw / iw etc. (Ops.cs:472-479)
  const float wr = __fdiv_rn((float)mw, (float)W), hr = __fdiv_rn((float)mh, (float)H);
  const float x1 = __fmul_rn(d[0], wr), x2 = __fmul_rn(d[2], wr);
  const float y1 = __fmul_rn(d[1], hr), y2 = __fmul_rn(d[3], hr);
  // crop_mask (Ops.cs:439-447) zeroes everything outside [x1,x2) x [y1,y2): only the box region needs
  // the coeff . proto dot products (typically a few % of the 160x160 map)
  for (int i = threadIdx.x; i < mh * mw; i += blockDim.x) mk_smem[i] = 0.f;
  const int cx0 = max(0, (int)ceilf(x1)), cx1 = min(mw, (int)ceilf(x2));  // c >= x1 && c < x2
  const int cy0 = max(0, (int)ceilf(y1)), cy1 = min(mh, (int)ceilf(y2));
  const int bw = max(0, cx1 - cx0), bh = max(0, cy1 - cy0);
  __syncthreads();
  for (int j = threadIdx.x; j < bw * bh; j += blockDim.x) {
    const int r = cy0 + j / bw, c = cx0 + j % bw;
    const int i = r * mw + c;
    float acc = 0.f;
    for (int k = 0; k < nm; k++) acc = fmaf(d[6 + k], pr[(size_t)k * mh * mw + i], acc);
    const bool inside = ((float)c >= x1) && ((float)c < x2) && ((float)r >= y1) && ((float)r < y2);
    mk_smem[i] = inside ? acc : 0.f;
  }
  __syncthreads();
  // ATen upsample_bilinear2d, align_corners=false: src = max(0, (dst + 0.5) * scale - 0.5),
  // scale = in/out
  const float sh = (float)mh / (float)H, sw = (float)mw / (float)W;
  uint8_t* out = masks + ((size_t)b * mask_cap + det) * H * W;
  // 4 consecutive pixels per thread -> one 32-bit store (the output, n x H x W bytes, is the HBM traffic)
  const int W4 = W >> 2;
  for (int i = threadIdx.x; i < H * W4; i += blockDim.x) {
    const int oy = i / W4, ox0 = (i - oy * W4) * 4;
    const float fy = fmaxf(0.f, ((float)oy + 0.5f) * sh - 0.5f);
    const int y0 = (int)fy;
    const int y1i = y0 + (y0 < mh - 1 ? 1 : 0);
    const float ly = fy - (float)y0, hy = 1.f - ly;
    uint32_t packed = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const float fx = fmaxf(0.f, ((float)(ox0 + j) + 0.5f) * sw - 0.5f);
      const int x0 = (int)fx;
      const int x1i = x0 + (x0 < mw - 1 ? 1 : 0);
      const float lx = fx - (float)x0, hx = 1.f - lx;
      const float v = hy * (hx * mk_smem[y0 * mw + x0] + lx * mk_smem[y0 * mw + x1i]) +
                      ly * (hx * mk_smem[y1i * mw + x0] + lx * mk_smem[y1i * mw + x1i]);
      packed |= (v > 0.f ? 1u : 0u) << (8 * j);
    }
    *reinterpret_cast<uint32_t*>(out + (size_t)oy * W + ox0) = packed;
  }
  for (int i = threadIdx.x; i < H * (W & 3); i += blockDim.x) {  // ragged right edge (W % 4 != 0)
    const int oy = i / (W & 3), ox = (W & ~3) + i % (W & 3);
    const float fy = fmaxf(0.f, ((float)oy + 0.5f) * sh - 0.5f), fx = fmaxf(0.f, ((float)ox + 0.5f) * sw - 0.5f);
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1i = y0 + (y0 < mh - 1 ? 1 : 0), x1i = x0 + (x0 < mw - 1 ? 1 : 0);
    const float ly = fy - (float)y0, lx = fx - (float)x0, hy = 1.f - ly, hx = 1.f - lx;
    const float v = hy * (hx * mk_smem[y0 * mw + x0] + lx * mk_smem[y0 * mw + x1i]) +
                    ly * (hx * mk_smem[y1i * mw + x0] + lx * mk_smem[y1i * mw + x1i]);
    out[(size_t)oy * W + ox] = v > 0.f ? 1 : 0;
  }
}

int masks_launch(const float* proto, const float* dets, const int* counts, int B, int max_det, int nm,
                 int mh, int mw, int H, int W, uint8_t* masks, cudaStream_t s, int mask_cap) {
  const size_t smem = (size_t)mh * mw * sizeof(float);
  if (smem > 200 * 1024) {
    set_error("yb_masks: proto map too large");
    return YB_ERR_SHAPE;
  }
  YB_CUDA_CHECK(smem_limit((const void*)masks_kernel, smem, false));
  if (mask_cap <= 0 || mask_cap > max_det) mask_cap = max_det;
  masks_kernel<<<dim3(mask_cap, B), 512, smem, s>>>(proto, dets, counts, max_det, mask_cap, nm, mh, mw, H, W, masks);
  YB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace yb
