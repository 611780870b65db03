// yb_train_step: the reference's whole training step behind ONE C-ABI call.
//
// Replaces `AMPWrapper.TrainStep` (Utils/Amp.cs:260-286: forward -> loss -> backward -> optimizer step) for the YOLOv8 and
// YOLOv11 detect models (graph wiring Models/Yolo.cs:45-134, 202-257; blocks Modules/Block.cs; head Modules/Head.cs:8-236):
// train-mode forward with batch-statistics BatchNorm, v8DetectionLoss (csrc/loss.cu), backward through the whole graph,
// AdamW over flat parameter buffers.  The graph walk that `yolosharp_b200/train.py` / `train_v11.py` do in Python over
// the library's kernels lives here in C++ over the same kernels (the Python steps stay as the executable specification
// this file is tested against, tests/test_trainer_native.py):
//   dense convolutions   TF32 tensor-core forward / dgrad / wgrad (csrc/conv_tf32.cu); the 3-channel stem runs with its
//                        input zero-padded to 8 channels
//   BatchNorm + SiLU     csrc/bn_train.cu (batch statistics, running-stat update, backward)
//   depthwise 3x3        csrc/train_v11.cu
//   attention core       csrc/attention.cu
//   everything between   small kernels below: channel-slice copies (concat / chunk), adds, nearest-2x upsample and its
//                        backward, MaxPool2d(5,1,2) with saved argmax and a gather-form (deterministic) backward, the
//                        NHWC <-> (B, C, A) head transposes, per-channel sums for the conv biases
// Memory: the caller owns the flat fp32 buffers (parameters, gradients, Adam moments, BatchNorm running statistics) - a
// data-parallel host all-reduces the gradient buffer between yb_train_backward and yb_train_apply; activations and
// gradients of a step live in one arena that is reset per step.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "common.cuh"

namespace yb {

namespace ts {

// ---------------------------------------------------------------------------------------------------------------
// small kernels
// ---------------------------------------------------------------------------------------------------------------
// dst[r, dcoff + c] (+)= src[r, scoff + c] for c < C: concat / chunk of NHWC tensors as channel-slice copies
__global__ void slice_copy_kernel(float* __restrict__ dst, int dpitch, int dcoff, const float* __restrict__ src, int spitch, int scoff,
                                  long long rows, int C, int accumulate) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * C) return;
  const long long r = i / C;
  const int c = (int)(i - r * C);
  const float v = src[r * spitch + scoff + c];
  float* d = dst + r * dpitch + dcoff + c;
  *d = accumulate ? *d + v : v;
}
// out = a + b on channel-slice views (row pitches may differ)
__global__ void add_kernel(float* __restrict__ out, int opitch, const float* __restrict__ a, int apitch, const float* __restrict__ b,
                           int bpitch, long long rows, int C) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * C) return;
  const long long r = i / C;
  const int c = (int)(i - r * C);
  out[r * opitch + c] = a[r * apitch + c] + b[r * bpitch + c];
}
// 4 channels per thread (C, pitches, channel offsets multiples of 4, 16-byte aligned bases; 32-bit index math): the scalar
// kernels above pay a 64-bit division per element
__global__ void slice_copy4_kernel(float* __restrict__ dst, int dpitch, const float* __restrict__ src, int spitch, int total4, int C4,
                                   int accumulate) {
  pdl_wait();
  pdl_trigger();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total4) return;
  const int r = i / C4, c = (i - r * C4) * 4;
  float4 v = *reinterpret_cast<const float4*>(src + (size_t)r * spitch + c);
  float4* d = reinterpret_cast<float4*>(dst + (size_t)r * dpitch + c);
  if (accumulate) { const float4 o = *d; v.x = o.x + v.x; v.y = o.y + v.y; v.z = o.z + v.z; v.w = o.w + v.w; }
  *d = v;
}
__global__ void add4_kernel(float* __restrict__ out, int opitch, const float* __restrict__ a, int apitch, const float* __restrict__ b,
                            int bpitch, int total4, int C4) {
  pdl_wait();
  pdl_trigger();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total4) return;
  const int r = i / C4, c = (i - r * C4) * 4;
  const float4 u = *reinterpret_cast<const float4*>(a + (size_t)r * apitch + c);
  const float4 v = *reinterpret_cast<const float4*>(b + (size_t)r * bpitch + c);
  *reinterpret_cast<float4*>(out + (size_t)r * opitch + c) = make_float4(u.x + v.x, u.y + v.y, u.z + v.z, u.w + v.w);
}
// nearest 2x upsample (Yolo.cs:70-84 `Upsample(scale_factor: 2)`), NHWC
__global__ void up2_forward_kernel(const float* __restrict__ x, int xpitch, float* __restrict__ y, int ypitch, int N, int H, int W, int C) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long n = (long long)N * 2 * H * 2 * W * C;
  if (i >= n) return;
  const int c = (int)(i % C);
  const long long po = i / C;
  long long p = po;
  const int wo = (int)(p % (2 * W)); p /= 2 * W;
  const int ho = (int)(p % (2 * H));
  const int b = (int)(p / (2 * H));
  y[po * ypitch + c] = x[(((long long)b * H + ho / 2) * W + wo / 2) * xpitch + c];
}
__global__ void up2_backward_kernel(const float* __restrict__ dy, int dpitch, float* __restrict__ dx, int N, int H, int W, int C) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long n = (long long)N * H * W * C;
  if (i >= n) return;
  const int c = (int)(i % C);
  long long p = i / C;
  const int w = (int)(p % W); p /= W;
  const int h = (int)(p % H);
  const int b = (int)(p / H);
  const float* r0 = dy + (((long long)b * 2 * H + 2 * h) * 2 * W + 2 * w) * dpitch + c;
  const float* r1 = r0 + (long long)2 * W * dpitch;
  // the 2 x 2 block summed sequentially in row-major order: the order of ATen's `sum((2, 4))` on the reshaped tensor.  (A
  // pairwise sum differs in the last bit of a few elements; through ~25 TF32 layers of backward that grew to 1e-3 of the
  // flat gradient - tools/dbg_native_determinism.py - so the order is part of the specification.)
  dx[i] = ((r0[0] + r0[dpitch]) + r1[0]) + r1[dpitch];  // the 2 x 2 block in row-major order, as `sum((2, 4))` of the reshaped tensor
}
// MaxPool2d(5, 1, 2) (Block.cs:275-279), NHWC, -inf padding; idx = flattened input position h * W + w of the maximum
// (first maximum in (kh, kw) scan order, as ATen's max_pool2d_with_indices)
__global__ void pool5_forward_kernel(const float* __restrict__ x, int xpitch, float* __restrict__ y, int ypitch, int* __restrict__ idx, int N,
                                     int H, int W, int C) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long n = (long long)N * H * W * C;
  if (i >= n) return;
  const int c = (int)(i % C);
  long long p = i / C;
  const int w = (int)(p % W); p /= W;
  const int h = (int)(p % H);
  const int b = (int)(p / H);
  float m = -INFINITY;
  int mi = -1;
  for (int dh = -2; dh <= 2; dh++) {
    const int hh = h + dh;
    if (hh < 0 || hh >= H) continue;
    for (int dw = -2; dw <= 2; dw++) {
      const int ww = w + dw;
      if (ww < 0 || ww >= W) continue;
      const float v = x[(((long long)b * H + hh) * W + ww) * xpitch + c];
      if (v > m || mi < 0 || v != v) { m = v; mi = hh * W + ww; }
    }
  }
  y[(i / C) * ypitch + c] = m;
  idx[i] = mi;
}
// backward as a gather: input position (h, w) receives the gradient of every output in its 5 x 5 neighbourhood whose
// argmax it is, summed in (dh, dw) order - deterministic, no atomics
__global__ void pool5_backward_kernel(const float* __restrict__ dy, int dpitch, const int* __restrict__ idx, float* __restrict__ dx, int N,
                                      int H, int W, int C) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long n = (long long)N * H * W * C;
  if (i >= n) return;
  const int c = (int)(i % C);
  long long p = i / C;
  const int w = (int)(p % W); p /= W;
  const int h = (int)(p % H);
  const int b = (int)(p / H);
  const int me = h * W + w;
  float acc = 0.f;
  for (int dh = -2; dh <= 2; dh++) {
    const int hh = h + dh;
    if (hh < 0 || hh >= H) continue;
    for (int dw = -2; dw <= 2; dw++) {
      const int ww = w + dw;
      if (ww < 0 || ww >= W) continue;
      const long long o = ((long long)b * H + hh) * W + ww;
      if (idx[o * C + c] == me) acc += dy[o * dpitch + c];
    }
  }
  dx[i] = acc;
}
// head: NHWC (B, h, w, C) -> out (B, C, A) at anchors [a0, a0 + h*w) (`view(b, c, -1)` + cat over levels, Head.cs:71-87)
__global__ void nhwc_to_bca_kernel(const float* __restrict__ x, float* __restrict__ out, int B, int HW, int C, int A, int a0) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * HW * C) return;
  const int a = (int)(i % HW);
  long long p = i / HW;
  const int c = (int)(p % C);
  const int b = (int)(p / C);
  out[((long long)b * C + c) * A + a0 + a] = x[((long long)b * HW + a) * C + c];
}
__global__ void bca_to_nhwc_kernel(const float* __restrict__ g, float* __restrict__ out, int B, int HW, int C, int A, int a0) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * HW * C) return;
  const int c = (int)(i % C);
  long long p = i / C;
  const int a = (int)(p % HW);
  const int b = (int)(p / HW);
  out[i] = g[((long long)b * C + c) * A + a0 + a];
}
// per-channel sum over rows (bias gradient of the plain Conv2d layers): slabs of 256 rows, partials folded in order
__global__ void colsum_partial_kernel(const float* __restrict__ x, long long rows, int C, float* __restrict__ part) {
  const int c = blockIdx.x * 32 + threadIdx.x;
  const long long r0 = (long long)blockIdx.y * 256;
  float a = 0.f;
  if (c < C)
    for (long long r = r0 + threadIdx.y; r < min(rows, r0 + 256); r += 8) a += x[r * C + c];
  __shared__ float s[8][32];
  s[threadIdx.y][threadIdx.x] = a;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    float t = 0.f;
    for (int k = 0; k < 8; k++) t += s[k][threadIdx.x];
    part[(size_t)blockIdx.y * C + c] = t;
  }
}
__global__ void colsum_fold_kernel(const float* __restrict__ part, int slabs, int C, float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float t = 0.f;
  for (int s = 0; s < slabs; s++) t += part[(size_t)s * C + c];
  out[c] = t;
}
// images (B, 3, H, W) NCHW u8 or f32 -> NHWC fp32 with the channels zero-padded to 8.  u8 pixels are scaled the way the
// training loader does it, `img.mul(1 / 255.0f)` (Data/YoloDataset.cs:140): a multiply by the rounded reciprocal, which is
// also what torch's CUDA `x / 255` computes; a true division differs by one ulp on ~40% of the pixel values.
__global__ void images_to_nhwc8_kernel(const void* __restrict__ in, int is_u8, float* __restrict__ out, int B, int H, int W) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long n = (long long)B * H * W;
  if (i >= n) return;
  const long long hw = (long long)H * W;
  const int b = (int)(i / hw);
  const long long p = i - (long long)b * hw;
  float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int c = 0; c < 3; c++) {
    const long long src = ((long long)b * 3 + c) * hw + p;
    v[c] = is_u8 ? (float)reinterpret_cast<const uint8_t*>(in)[src] * (1.0f / 255.0f) : reinterpret_cast<const float*>(in)[src];
  }
  float4* o = reinterpret_cast<float4*>(out + i * 8);
  o[0] = make_float4(v[0], v[1], v[2], v[3]);
  o[1] = make_float4(0.f, 0.f, 0.f, 0.f);
}
// weight (Cout, 3, k, k) -> (Cout, 8, k, k) zero padded; gradient back: the first 3 input channels
__global__ void pad_weight8_kernel(const float* __restrict__ w, float* __restrict__ w8, int Cout, int kk) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Cout * 8 * kk) return;
  const int t = i % kk, ci = (i / kk) % 8, co = i / (8 * kk);
  w8[i] = ci < 3 ? w[(co * 3 + ci) * kk + t] : 0.f;
}
__global__ void unpad_weight8_kernel(const float* __restrict__ g8, float* __restrict__ g, int Cout, int kk) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Cout * 3 * kk) return;
  const int t = i % kk, ci = (i / kk) % 3, co = i / (3 * kk);
  g[i] = g8[(co * 8 + ci) * kk + t];
}

static inline unsigned nb(long long n, int t = 256) { return (unsigned)((n + t - 1) / t); }

// ---------------------------------------------------------------------------------------------------------------
// tensors, arena, parameters
// ---------------------------------------------------------------------------------------------------------------
// NHWC tensor or a channel-slice VIEW of one: element (n, h, w, c) at p[((n*H + h)*W + w) * pitch + c].  Views replace the
// chunk / cat copies of the graph (Block.cs:391-396): producers write their slice of the concat buffer, consumers read theirs.
struct T4 {
  float* p = nullptr;
  int N = 0, H = 0, W = 0, C = 0, pitch = 0;
  long long rows() const { return (long long)N * H * W; }
  long long numel() const { return rows() * C; }
  bool dense() const { return pitch == C; }
};
static T4 view(const T4& t, int c0, int C) {
  T4 v = t;
  v.p = t.p + c0;
  v.C = C;
  return v;
}

struct Entry { std::string name; std::vector<int64_t> shape; long long off = 0, count = 0; int kind = 0; };  // kind 0 parameter, 1 running stat

struct Net {
  int arch = 8, size = 0, nc = 80, reg_max = 16, max_batch = 1, H = 640, W = 640;
  cudaStream_t s = nullptr;
  std::vector<Entry> params, stats;                 // order = layout of the flat buffers (bias group first)
  std::map<std::string, int> pidx, sidx;
  float *P = nullptr, *G = nullptr, *M1 = nullptr, *M2 = nullptr, *R = nullptr;  // caller-owned flat buffers
  long long n_params = 0, n_bias = 0, n_stats = 0;
  char* arena = nullptr;
  size_t arena_cap = 0, arena_off = 0;
  float* ws = nullptr;
  size_t ws_bytes = 0;
  // tensor-core operand layouts of every dense conv weight, same offsets as P; repacked once per step (tf_pack_all)
  float *WF = nullptr, *WB = nullptr;
  unsigned* bn_counters = nullptr;  // 64 zeroed tickets of the BatchNorm statistics kernels (they leave them zero; one stream)
  TfPackDesc* pack_descs = nullptr;
  int n_packs = 0;
  long long pack_chunks = 0;
  int step_count = 0;
  int rc = 0;  // first error of the current step (modules return empty tensors after it)
  // eval mode (yb_trainer_evaluate): BatchNorm on the running statistics, folded by ONE launch per forward into EV, a
  // parameter-sized buffer laid out like P: a dense conv's folded [tap][Cout][Cin] operand at its weight's offset, the folded
  // bias at its bn.bias offset, 1 / sqrt(rv + eps) at its bn.weight offset (read by the stem and depthwise convs, whose
  // BatchNorm stays a separate pass); the head's plain Conv2d weights packed unscaled at their offset
  bool eval = false;
  float* EV = nullptr;
  TfFoldDesc* fold_descs = nullptr;
  int n_folds = 0;
  long long fold_chunks = 0;

  float* alloc(long long n) {
    const size_t bytes = ((size_t)n * sizeof(float) + 255) & ~(size_t)255;
    if (arena_off + bytes > arena_cap) { if (!rc) { rc = YB_ERR_STATE; set_error("yb_train_step: activation arena exhausted"); } return nullptr; }
    float* p = reinterpret_cast<float*>(arena + arena_off);
    arena_off += bytes;
    return p;
  }
  T4 make(int N_, int H_, int W_, int C_) {
    T4 t; t.N = N_; t.H = H_; t.W = W_; t.C = C_; t.pitch = C_;
    t.p = alloc(t.numel());
    return t;
  }
  float* p(const std::string& k) { return P + params[pidx.at(k)].off; }
  const float* wf(const std::string& k) { return WF ? WF + params[pidx.at(k)].off : nullptr; }
  const float* wb(const std::string& k) { return WB ? WB + params[pidx.at(k)].off : nullptr; }
  float* g(const std::string& k) { return G + params[pidx.at(k)].off; }
  float* r(const std::string& k) { return R + stats[sidx.at(k)].off; }
  float* ev(const std::string& k) { return EV + params[pidx.at(k)].off; }
  void check(int code) { if (code && !rc) rc = code; }
  void check_launch() { if (!rc && cudaGetLastError() != cudaSuccess) { rc = YB_ERR_CUDA; set_error("yb_train_step: kernel launch failed"); } }
};

static bool vec4_ok(long long numel, int C, const void* p0, int pitch0, const void* p1, int pitch1, const void* p2, int pitch2) {
  return C % 4 == 0 && pitch0 % 4 == 0 && pitch1 % 4 == 0 && pitch2 % 4 == 0 && numel / 4 < (1ll << 31) &&
         (((uintptr_t)p0 | (uintptr_t)p1 | (uintptr_t)p2) & 15) == 0;
}
static void put(Net& n, const T4& dst, int c0, const T4& src, bool accumulate = false) {  // dst[..., c0 : c0 + src.C] (+)= src
  if (n.rc) return;
  if (vec4_ok(src.numel(), src.C, dst.p + c0, dst.pitch, src.p, src.pitch, src.p, src.pitch))
    n.check(launch_pdl(slice_copy4_kernel, dim3(nb(src.numel() / 4)), dim3(256), 0, n.s, dst.p + c0, dst.pitch, (const float*)src.p, src.pitch,
                       (int)(src.numel() / 4), src.C / 4, accumulate ? 1 : 0) == cudaSuccess ? 0 : YB_ERR_CUDA);
  else
    slice_copy_kernel<<<nb(src.numel()), 256, 0, n.s>>>(dst.p, dst.pitch, c0, src.p, src.pitch, 0, src.rows(), src.C, accumulate ? 1 : 0);
  n.check_launch();
}
static T4 dense_copy(Net& n, const T4& x) {  // contiguous copy of a view (kernels that take no pitch)
  if (x.dense()) return x;
  T4 y = n.make(x.N, x.H, x.W, x.C);
  put(n, y, 0, x);
  return y;
}
static void add_into(Net& n, const T4& out, const T4& a, const T4& b) {
  if (n.rc) return;
  if (vec4_ok(a.numel(), a.C, out.p, out.pitch, a.p, a.pitch, b.p, b.pitch))
    n.check(launch_pdl(add4_kernel, dim3(nb(a.numel() / 4)), dim3(256), 0, n.s, out.p, out.pitch, (const float*)a.p, a.pitch, (const float*)b.p,
                       b.pitch, (int)(a.numel() / 4), a.C / 4) == cudaSuccess ? 0 : YB_ERR_CUDA);
  else
    add_kernel<<<nb(a.numel()), 256, 0, n.s>>>(out.p, out.pitch, a.p, a.pitch, b.p, b.pitch, a.rows(), a.C);
  n.check_launch();
}
static T4 add(Net& n, const T4& a, const T4& b) {
  T4 y = n.make(a.N, a.H, a.W, a.C);
  add_into(n, y, a, b);
  return y;
}

// ---------------------------------------------------------------------------------------------------------------
// modules (forward saves what backward needs; one forward per step)
// ---------------------------------------------------------------------------------------------------------------
// forward(x, dst): x may be a view; when dst is given the module writes its output there (a slice of its consumer's concat
// buffer) and returns it.  backward(dy): dy may be a view; the result is a dense tensor.
struct Module {
  virtual ~Module() {}
  virtual T4 forward(Net& n, T4 x, const T4* dst = nullptr) = 0;
  virtual T4 backward(Net& n, T4 dy) = 0;
};
typedef std::unique_ptr<Module> Mod;

// Conv block: Conv2d(bias: false) -> BatchNorm2d(train) -> SiLU / identity (Convs.cs:36-56); groups > 1 = depthwise 3x3
struct Conv : Module {
  std::string name;
  int cin, cout, k, s, act, depthwise;
  bool need_dx = true, pad8 = false;
  T4 x, z;
  float *mean = nullptr, *invstd = nullptr;
  Conv(Net& n, const std::string& nm, int cin_, int cout_, int k_, int s_ = 1, bool act_ = true, bool dw = false)
      : name(nm), cin(cin_), cout(cout_), k(k_), s(s_), act(act_ ? 1 : 0), depthwise(dw ? 1 : 0) {
    (void)n;
  }
  T4 forward(Net& n, T4 in, const T4* dst = nullptr) override {
    if (n.eval) return forward_eval(n, in, dst, nullptr);
    x = depthwise ? dense_copy(n, in) : in;  // the depthwise kernels take dense tensors
    const int Ho = (in.H + 2 * (k / 2) - k) / s + 1, Wo = (in.W + 2 * (k / 2) - k) / s + 1;
    z = n.make(in.N, Ho, Wo, cout);
    T4 y = dst ? *dst : n.make(in.N, Ho, Wo, cout);
    mean = n.alloc(cout);
    invstd = n.alloc(cout);
    if (n.rc) return y;
    const float* w = n.p(name + ".conv.weight");
    if (depthwise) {
      n.check(dwconv3x3_forward_f32(x.p, w, x.N, x.H, x.W, x.C, z.p, n.s));
    } else if (pad8 && k == 3 && s == 2 && cout % 8 == 0 && cout <= 128) {
      n.check(stem3_forward(x.p, 8, w, x.N, x.H, x.W, cout, z.p, n.s));  // the 3-channel stem: fp32 CUDA cores (conv_tf32.cu)
    } else if (pad8) {
      float* w8 = n.alloc((long long)cout * 8 * k * k);
      if (n.rc) return y;
      pad_weight8_kernel<<<nb((long long)cout * 8 * k * k), 256, 0, n.s>>>(w, w8, cout, k * k);
      n.check(tf_conv_forward(x.p, w8, nullptr, x.N, x.H, x.W, 8, cout, k, s, k / 2, z.p, n.ws, n.ws_bytes, n.s, 0, nullptr));
    } else {
      n.check(tf_conv_forward(x.p, w, nullptr, x.N, x.H, x.W, cin, cout, k, s, k / 2, z.p, n.ws, n.ws_bytes, n.s, x.dense() ? 0 : x.pitch,
                              n.wf(name + ".conv.weight")));
    }
    n.check(bn_silu_train_forward(z.p, z.rows(), cout, cout, n.p(name + ".bn.weight"), n.p(name + ".bn.bias"), 1e-3f, 0.03f, act,
                                  n.r(name + ".bn.running_mean"), n.r(name + ".bn.running_var"), y.p, y.pitch, mean, invstd, n.s, n.bn_counters));
    return y;
  }
  // eval mode (Convs.cs:36-56 in `eval()`): a dense conv is ONE launch on the folded operands, + res after the activation
  // when given; the stem and depthwise convs keep their forward kernel and apply BatchNorm with the running statistics
  T4 forward_eval(Net& n, T4 in, const T4* dst, const T4* res) {
    const int Ho = (in.H + 2 * (k / 2) - k) / s + 1, Wo = (in.W + 2 * (k / 2) - k) / s + 1;
    T4 y = dst ? *dst : n.make(in.N, Ho, Wo, cout);
    if (n.rc) return y;
    const bool stem = pad8 && k == 3 && s == 2 && cout % 8 == 0 && cout <= 128;
    if (!depthwise && !stem) {
      if (pad8) { n.check(YB_ERR_SHAPE); set_error("yb_trainer_evaluate: the stem needs cout % 8 == 0 and cout <= 128"); return y; }
      n.check(tf_conv_forward_eval(in.p, in.pitch, n.ev(name + ".conv.weight"), n.ev(name + ".bn.bias"), in.N, in.H, in.W, cin, cout, k, s,
                                   act, res ? res->p : nullptr, res ? res->pitch : 0, y.p, y.pitch, 0, n.s));
      return y;
    }
    const T4 xin = depthwise ? dense_copy(n, in) : in;
    T4 zz = n.make(in.N, Ho, Wo, cout);
    if (n.rc) return y;
    const float* w = n.p(name + ".conv.weight");
    if (depthwise) n.check(dwconv3x3_forward_f32(xin.p, w, xin.N, xin.H, xin.W, xin.C, zz.p, n.s));
    else n.check(stem3_forward(xin.p, 8, w, xin.N, xin.H, xin.W, cout, zz.p, n.s));
    n.check(bn_silu_apply(zz.p, zz.rows(), cout, cout, n.r(name + ".bn.running_mean"), n.ev(name + ".bn.weight"), n.p(name + ".bn.weight"),
                          n.p(name + ".bn.bias"), act, y.p, y.pitch, n.s));
    return y;
  }
  T4 backward(Net& n, T4 dy) override {
    T4 dz = n.make(z.N, z.H, z.W, z.C);
    T4 dx;
    if (n.rc) return dx;
    n.check(bn_silu_backward(z.p, dy.p, z.rows(), cout, cout, dy.pitch, n.p(name + ".bn.weight"), n.p(name + ".bn.bias"), mean, invstd, act,
                             dz.p, cout, n.g(name + ".bn.weight"), n.g(name + ".bn.bias"), n.s, n.bn_counters));
    const float* w = n.p(name + ".conv.weight");
    float* gw = n.g(name + ".conv.weight");
    if (depthwise) {
      dx = n.make(x.N, x.H, x.W, x.C);
      if (n.rc) return dx;
      n.check(dwconv3x3_backward_f32(x.p, dz.p, w, x.N, x.H, x.W, x.C, dx.p, gw, n.s));
    } else if (pad8 && k == 3 && s == 2 && cout % 8 == 0 && cout <= 128) {
      n.check(stem3_backward_weight(x.p, 8, dz.p, x.N, x.H, x.W, cout, gw, n.ws, n.ws_bytes, n.s));  // the images need no gradient
    } else if (pad8) {
      float* g8 = n.alloc((long long)cout * 8 * k * k);
      if (n.rc) return dx;
      n.check(tf_conv_backward_weight(x.p, dz.p, x.N, x.H, x.W, 8, cout, k, s, k / 2, g8, n.ws, n.ws_bytes, n.s, 0));
      unpad_weight8_kernel<<<nb((long long)cout * 3 * k * k), 256, 0, n.s>>>(g8, gw, cout, k * k);
      n.check_launch();  // the images need no gradient
    } else {
      if (need_dx) {
        dx = n.make(x.N, x.H, x.W, x.C);
        if (n.rc) return dx;
        n.check(tf_conv_backward_data(dz.p, w, x.N, x.H, x.W, cin, cout, k, s, k / 2, dx.p, n.ws, n.ws_bytes, n.s, n.wb(name + ".conv.weight")));
      }
      n.check(tf_conv_backward_weight(x.p, dz.p, x.N, x.H, x.W, cin, cout, k, s, k / 2, gw, n.ws, n.ws_bytes, n.s, x.dense() ? 0 : x.pitch));
    }
    return dx;
  }
};

// plain Conv2d(k = 1, bias: true): the last layer of every Detect branch (Head.cs:41-52)
struct Conv2dBias : Module {
  std::string name;
  int cin, cout;
  T4 x;
  Conv2dBias(const std::string& nm, int cin_, int cout_) : name(nm), cin(cin_), cout(cout_) {}
  T4 forward(Net& n, T4 in, const T4* dst = nullptr) override {
    (void)dst;  // the head outputs are transposed into (B, C, A) by the caller
    x = in;
    T4 y = n.make(in.N, in.H, in.W, cout);
    if (n.rc) return y;
    if (n.eval) {  // the packed weights of the step (WF) may predate the last optimizer step: EV holds the current ones
      n.check(tf_conv_forward_eval(in.p, in.pitch, n.ev(name + ".weight"), n.p(name + ".bias"), in.N, in.H, in.W, cin, cout, 1, 1, 0, nullptr, 0,
                                   y.p, y.pitch, 0, n.s));
      return y;
    }
    n.check(tf_conv_forward(in.p, n.p(name + ".weight"), n.p(name + ".bias"), in.N, in.H, in.W, cin, cout, 1, 1, 0, y.p, n.ws, n.ws_bytes, n.s,
                            in.dense() ? 0 : in.pitch, n.wf(name + ".weight")));
    return y;
  }
  T4 backward(Net& n, T4 dz_in) override {
    T4 dz = dense_copy(n, dz_in);
    T4 dx = n.make(x.N, x.H, x.W, x.C);
    if (n.rc) return dx;
    n.check(tf_conv_backward_data(dz.p, n.p(name + ".weight"), x.N, x.H, x.W, cin, cout, 1, 1, 0, dx.p, n.ws, n.ws_bytes, n.s,
                                  n.wb(name + ".weight")));
    n.check(tf_conv_backward_weight(x.p, dz.p, x.N, x.H, x.W, cin, cout, 1, 1, 0, n.g(name + ".weight"), n.ws, n.ws_bytes, n.s,
                                    x.dense() ? 0 : x.pitch));
    const long long rows = dz.rows();
    const int slabs = (int)((rows + 255) / 256);
    float* part = n.alloc((long long)slabs * cout);
    if (n.rc) return dx;
    colsum_partial_kernel<<<dim3((cout + 31) / 32, slabs), dim3(32, 8), 0, n.s>>>(dz.p, rows, cout, part);
    colsum_fold_kernel<<<(cout + 127) / 128, 128, 0, n.s>>>(part, slabs, cout, n.g(name + ".bias"));
    n.check_launch();
    return dx;
  }
};

struct Seq : Module {
  std::vector<Mod> layers;
  T4 forward(Net& n, T4 x, const T4* dst = nullptr) override {
    for (size_t i = 0; i < layers.size(); i++) x = layers[i]->forward(n, x, i + 1 == layers.size() ? dst : nullptr);
    return x;
  }
  T4 backward(Net& n, T4 d) override { for (size_t i = layers.size(); i-- > 0;) d = layers[i]->backward(n, d); return d; }
};

// Bottleneck (Block.cs:572-607), k = (3, 3)
struct Bottleneck : Module {
  Conv cv1, cv2;
  bool add_;
  Bottleneck(Net& n, const std::string& nm, int c1, int c2, bool shortcut, double e)
      : cv1(n, nm + ".cv1", c1, (int)(c2 * e), 3), cv2(n, nm + ".cv2", (int)(c2 * e), c2, 3), add_(shortcut && c1 == c2) {}
  T4 forward(Net& n, T4 x, const T4* dst = nullptr) override {
    if (!add_) return cv2.forward(n, cv1.forward(n, x), dst);
    if (n.eval) return cv2.forward_eval(n, cv1.forward(n, x), dst, &x);  // the shortcut add in cv2's epilogue
    T4 y = cv2.forward(n, cv1.forward(n, x));
    T4 out = dst ? *dst : n.make(x.N, x.H, x.W, x.C);
    add_into(n, out, x, y);
    return out;
  }
  T4 backward(Net& n, T4 dy) override {
    T4 dx = cv1.backward(n, cv2.backward(n, dy));
    return add_ ? add(n, dx, dy) : dx;
  }
};

// C3k (Block.cs:404-441, 611-620): cv3(cat(m(cv1 x), cv2 x)), hidden = c2 / 2, n bottlenecks with e = 1
struct C3k : Module {
  Conv cv1, cv2, cv3;
  std::vector<Mod> m;
  int ch;
  C3k(Net& n, const std::string& nm, int c1, int c2, int reps, bool shortcut)
      : cv1(n, nm + ".cv1", c1, c2 / 2, 1), cv2(n, nm + ".cv2", c1, c2 / 2, 1), cv3(n, nm + ".cv3", 2 * (c2 / 2), c2, 1), ch(c2 / 2) {
    for (int i = 0; i < reps; i++) m.emplace_back(new Bottleneck(n, nm + ".m." + std::to_string(i), ch, ch, shortcut, 1.0));
  }
  T4 forward(Net& n, T4 x, const T4* dst = nullptr) override {
    T4 cat = n.make(x.N, x.H, x.W, 2 * ch);
    const T4 ca = view(cat, 0, ch), cb = view(cat, ch, ch);
    T4 a = cv1.forward(n, x, m.empty() ? &ca : nullptr);
    for (size_t i = 0; i < m.size(); i++) a = m[i]->forward(n, a, i + 1 == m.size() ? &ca : nullptr);
    cv2.forward(n, x, &cb);
    return cv3.forward(n, cat, dst);
  }
  T4 backward(Net& n, T4 dy) override {
    T4 d = cv3.backward(n, dy);
    T4 da = view(d, 0, ch);
    for (size_t i = m.size(); i-- > 0;) da = m[i]->backward(n, da);
    return add(n, cv1.backward(n, da), cv2.backward(n, view(d, ch, ch)));
  }
};

// C2f (Block.cs:371-398) and C3k2 (Block.cs:623-661): cv1 -> chunk 2 -> n inner blocks chained on the last chunk -> cat -> cv2
struct C2f : Module {
  Conv cv1, cv2;
  std::vector<Mod> m;
  int c;
  // inner: 0 = Bottleneck(c, c, shortcut, e = 1.0) (C2f), 1 = Bottleneck(c, c, shortcut, e = 0.5) (C3k2, c3k = false), 2 = C3k(c, c, 2, shortcut)
  C2f(Net& n, const std::string& nm, int c1, int c2, int reps, bool shortcut, double e, int inner)
      : cv1(n, nm + ".cv1", c1, 2 * (int)(c2 * e), 1), cv2(n, nm + ".cv2", (2 + reps) * (int)(c2 * e), c2, 1), c((int)(c2 * e)) {
    for (int i = 0; i < reps; i++) {
      const std::string mn = nm + ".m." + std::to_string(i);
      if (inner == 2) m.emplace_back(new C3k(n, mn, c, c, 2, shortcut));
      else m.emplace_back(new Bottleneck(n, mn, c, c, shortcut, inner == 0 ? 1.0 : 0.5));
    }
  }
  T4 forward(Net& n, T4 x, const T4* dst = nullptr) override {
    const int reps = (int)m.size();
    T4 cat = n.make(x.N, x.H, x.W, (2 + reps) * c);  // every producer writes its own slice: no chunk / cat copies
    const T4 y01 = view(cat, 0, 2 * c);
    cv1.forward(n, x, &y01);
    for (int i = 0; i < reps; i++) {
      const T4 out = view(cat, (2 + i) * c, c);
      m[i]->forward(n, view(cat, (1 + i) * c, c), &out);
    }
    return cv2.forward(n, cat, dst);
  }
  T4 backward(Net& n, T4 dy) override {
    T4 d = cv2.backward(n, dy);  // (2 + reps) c channels; slice i+1 accumulates the gradient coming back through block i
    const int reps = (int)m.size();
    for (int i = reps - 1; i >= 0; i--) put(n, d, (1 + i) * c, m[i]->backward(n, view(d, (2 + i) * c, c)), true);
    return cv1.backward(n, view(d, 0, 2 * c));
  }
};

// SPPF (Block.cs:236-282): cv1 has NO activation in the reference (:257)
struct SPPF : Module {
  Conv cv1, cv2;
  T4 t[4];
  int* idx[3] = {nullptr, nullptr, nullptr};
  int ch;
  SPPF(Net& n, const std::string& nm, int c1, int c2) : cv1(n, nm + ".cv1", c1, c1 / 2, 1, 1, false), cv2(n, nm + ".cv2", 4 * (c1 / 2), c2, 1), ch(c1 / 2) {}
  T4 forward(Net& n, T4 x, const T4* dst = nullptr) override {
    T4 cat = n.make(x.N, x.H, x.W, 4 * ch);
    for (int i = 0; i < 4; i++) t[i] = view(cat, i * ch, ch);
    cv1.forward(n, x, &t[0]);
    for (int i = 0; i < 3; i++) {
      idx[i] = reinterpret_cast<int*>(n.alloc(t[i].numel()));
      if (n.rc) return cat;
      pool5_forward_kernel<<<nb(t[i].numel()), 256, 0, n.s>>>(t[i].p, t[i].pitch, t[i + 1].p, t[i + 1].pitch, idx[i], x.N, x.H, x.W, ch);
      n.check_launch();
    }
    return cv2.forward(n, cat, dst);
  }
  T4 backward(Net& n, T4 dy) override {
    T4 d = cv2.backward(n, dy);
    for (int i = 2; i >= 0; i--) {
      const T4 up = view(d, (i + 1) * ch, ch);
      T4 pb = n.make(d.N, d.H, d.W, ch);
      if (n.rc) return pb;
      pool5_backward_kernel<<<nb(pb.numel()), 256, 0, n.s>>>(up.p, up.pitch, idx[i], pb.p, d.N, d.H, d.W, ch);
      n.check_launch();
      put(n, d, i * ch, pb, true);
    }
    return cv1.backward(n, view(d, 0, ch));
  }
};

// Attention (Block.cs:752-809), NHWC: qkv (B, H, W, nh * (2 kd + hd)) viewed per head as [q (kd) | k (kd) | v (hd)]
struct Attention : Module {
  Conv qkv, proj, pe;
  int nh, hd, kd, dim;
  float scale;
  T4 q, k, v;
  Attention(Net& n, const std::string& nm, int dim_, int heads)
      // qkv / proj / pe keep the Conv block's default SiLU in the reference (Block.cs:744-746 pass no `act: false`)
      : qkv(n, nm + ".qkv", dim_, dim_ + 2 * heads * (int)((dim_ / heads) * 0.5), 1, 1, true), proj(n, nm + ".proj", dim_, dim_, 1, 1, true),
        pe(n, nm + ".pe", dim_, dim_, 3, 1, true, true), nh(heads), hd(dim_ / heads), kd((int)((dim_ / heads) * 0.5)), dim(dim_),
        scale(1.0f / std::sqrt((float)(int)((dim_ / heads) * 0.5))) {}
  // split / merge of the per-head interleaved qkv tensor: token rows of nh groups [q | k | v]
  void split_qkv(Net& n, const T4& t) {
    const int per = 2 * kd + hd;
    const long long rows = t.rows() * nh;  // (token, head) rows of `per` channels
    q = n.make(t.N, t.H, t.W, nh * kd); k = n.make(t.N, t.H, t.W, nh * kd); v = n.make(t.N, t.H, t.W, nh * hd);
    if (n.rc) return;
    slice_copy_kernel<<<nb(rows * kd), 256, 0, n.s>>>(q.p, kd, 0, t.p, per, 0, rows, kd, 0);
    slice_copy_kernel<<<nb(rows * kd), 256, 0, n.s>>>(k.p, kd, 0, t.p, per, kd, rows, kd, 0);
    slice_copy_kernel<<<nb(rows * hd), 256, 0, n.s>>>(v.p, hd, 0, t.p, per, 2 * kd, rows, hd, 0);
    n.check_launch();
  }
  T4 forward(Net& n, T4 x, const T4* dst = nullptr) override {
    T4 t = qkv.forward(n, x);
    split_qkv(n, t);
    T4 o = n.make(x.N, x.H, x.W, dim);
    if (n.rc) return o;
    n.check(attention_forward_f32(q.p, k.p, v.p, x.N, x.H * x.W, nh, kd, hd, scale, o.p, nullptr, nullptr, n.s));
    T4 y = add(n, o, pe.forward(n, v));
    return proj.forward(n, y, dst);
  }
  T4 backward(Net& n, T4 dy) override {
    T4 d = proj.backward(n, dy);
    T4 dv_pe = pe.backward(n, d);
    T4 dq = n.make(q.N, q.H, q.W, q.C), dk = n.make(k.N, k.H, k.W, k.C), dv = n.make(v.N, v.H, v.W, v.C);
    const int per = 2 * kd + hd;
    T4 dqkv = n.make(d.N, d.H, d.W, nh * per);
    if (n.rc) return dqkv;
    n.check(attention_backward_f32(q.p, k.p, v.p, d.p, d.N, d.H * d.W, nh, kd, hd, scale, dq.p, dk.p, dv.p, n.s));
    T4 dvs = add(n, dv, dv_pe);
    if (n.rc) return dqkv;
    const long long rows = d.rows() * nh;
    slice_copy_kernel<<<nb(rows * kd), 256, 0, n.s>>>(dqkv.p, per, 0, dq.p, kd, 0, rows, kd, 0);
    slice_copy_kernel<<<nb(rows * kd), 256, 0, n.s>>>(dqkv.p, per, kd, dk.p, kd, 0, rows, kd, 0);
    slice_copy_kernel<<<nb(rows * hd), 256, 0, n.s>>>(dqkv.p, per, 2 * kd, dvs.p, hd, 0, rows, hd, 0);
    n.check_launch();
    return qkv.backward(n, dqkv);
  }
};

// PSABlock (Block.cs:697-722, shortcut = true)
struct PSABlock : Module {
  Attention attn;
  Conv f0, f1;
  PSABlock(Net& n, const std::string& nm, int c) : attn(n, nm + ".attn", c, c / 64), f0(n, nm + ".ffn.0", c, 2 * c, 1), f1(n, nm + ".ffn.1", 2 * c, c, 1) {}  // ffn[1] keeps its SiLU too (Block.cs:708)
  T4 forward(Net& n, T4 x, const T4* dst = nullptr) override {
    T4 a = add(n, x, attn.forward(n, x));
    T4 out = dst ? *dst : n.make(x.N, x.H, x.W, x.C);
    add_into(n, out, a, f1.forward(n, f0.forward(n, a)));
    return out;
  }
  T4 backward(Net& n, T4 dy) override {
    T4 d = add(n, dy, f0.backward(n, f1.backward(n, dy)));
    return add(n, d, attn.backward(n, d));
  }
};

// C2PSA (Block.cs:664-695)
struct C2PSA : Module {
  Conv cv1, cv2;
  std::vector<Mod> m;
  int c;
  C2PSA(Net& n, const std::string& nm, int c1, int reps) : cv1(n, nm + ".cv1", c1, 2 * (c1 / 2), 1), cv2(n, nm + ".cv2", 2 * (c1 / 2), c1, 1), c(c1 / 2) {
    for (int i = 0; i < reps; i++) m.emplace_back(new PSABlock(n, nm + ".m." + std::to_string(i), c));
  }
  T4 forward(Net& n, T4 x, const T4* dst = nullptr) override {
    T4 y = cv1.forward(n, x);
    T4 cat = n.make(x.N, x.H, x.W, 2 * c);  // a separate buffer: the blocks' convs keep views of y for their weight gradients
    put(n, cat, 0, view(y, 0, c));
    T4 b = view(y, c, c);
    const T4 cb = view(cat, c, c);
    for (size_t i = 0; i < m.size(); i++) b = m[i]->forward(n, b, i + 1 == m.size() ? &cb : nullptr);
    return cv2.forward(n, cat, dst);
  }
  T4 backward(Net& n, T4 dy) override {
    T4 d = cv2.backward(n, dy);
    T4 db = view(d, c, c);
    for (size_t i = m.size(); i-- > 0;) db = m[i]->backward(n, db);
    put(n, d, c, db);  // d = [da | db] again
    return cv1.backward(n, d);
  }
};

// Detect.forward_head (Head.cs:35-53, 71-87): per level a box branch and a class branch (legacy = the v8 branch of two
// 3x3 Convs; v11: DWConv + 1x1 Conv twice), outputs concatenated over levels as (B, C, A)
struct Detect {
  std::vector<Seq> cv2, cv3;
  int nc, reg_max;
  std::vector<T4> shapes;
  Detect(Net& n, const std::string& nm, int nc_, const int ch[3], bool legacy) : nc(nc_), reg_max(16) {
    const int c2 = std::max(16, std::max(ch[0] / 4, reg_max * 4)), c3 = std::max(ch[0], std::min(nc, 100));
    cv2.resize(3);
    cv3.resize(3);
    for (int i = 0; i < 3; i++) {
      const std::string b = nm + ".cv2." + std::to_string(i), c = nm + ".cv3." + std::to_string(i);
      cv2[i].layers.emplace_back(new Conv(n, b + ".0", ch[i], c2, 3));
      cv2[i].layers.emplace_back(new Conv(n, b + ".1", c2, c2, 3));
      cv2[i].layers.emplace_back(new Conv2dBias(b + ".2", c2, 4 * reg_max));
      if (legacy) {
        cv3[i].layers.emplace_back(new Conv(n, c + ".0", ch[i], c3, 3));
        cv3[i].layers.emplace_back(new Conv(n, c + ".1", c3, c3, 3));
      } else {
        cv3[i].layers.emplace_back(new Conv(n, c + ".0.0", ch[i], ch[i], 3, 1, true, true));
        cv3[i].layers.emplace_back(new Conv(n, c + ".0.1", ch[i], c3, 1));
        cv3[i].layers.emplace_back(new Conv(n, c + ".1.0", c3, c3, 3, 1, true, true));
        cv3[i].layers.emplace_back(new Conv(n, c + ".1.1", c3, c3, 1));
      }
      cv3[i].layers.emplace_back(new Conv2dBias(c + ".2", c3, nc));
    }
  }
  // boxes / scores: the raw outputs (B, C, A), each skipped when null (eval); pred: the decoded (B, 4 + nc, A) of the fp32
  // engine (`Detect._inference`, Head.cs:204-223), written when given
  void forward(Net& n, const T4 feats[3], float* boxes, float* scores, int A, float* pred = nullptr) {
    shapes.assign(feats, feats + 3);
    int a0 = 0;
    for (int i = 0; i < 3; i++) {
      T4 b = cv2[i].forward(n, feats[i]);
      T4 s = cv3[i].forward(n, feats[i]);
      if (n.rc) return;
      const int hw = feats[i].H * feats[i].W;
      if (boxes) nhwc_to_bca_kernel<<<nb((long long)b.N * hw * b.C), 256, 0, n.s>>>(b.p, boxes, b.N, hw, b.C, A, a0);
      if (scores) nhwc_to_bca_kernel<<<nb((long long)s.N * hw * s.C), 256, 0, n.s>>>(s.p, scores, s.N, hw, s.C, A, a0);
      n.check_launch();
      if (pred) {
        View vb, vc;
        vb.base = b.p; vb.H = b.H; vb.W = b.W; vb.pitch = b.pitch; vb.C = b.C;
        vc.base = s.p; vc.H = s.H; vc.W = s.W; vc.pitch = s.pitch; vc.C = s.C;
        n.check(launch_decode_level<float>(vb, vc, nullptr, b.N, nc, 0, reg_max, (float)(n.H / b.H), a0, A, 4 + nc, pred, n.s));
      }
      a0 += hw;
    }
  }
  void backward(Net& n, const float* gboxes, const float* gscores, int A, T4 out[3]) {
    int a0 = 0;
    for (int i = 0; i < 3; i++) {
      const T4& f = shapes[i];
      const int hw = f.H * f.W;
      T4 gb = n.make(f.N, f.H, f.W, 4 * reg_max), gs = n.make(f.N, f.H, f.W, nc);
      if (n.rc) return;
      bca_to_nhwc_kernel<<<nb(gb.numel()), 256, 0, n.s>>>(gboxes, gb.p, f.N, hw, 4 * reg_max, A, a0);
      bca_to_nhwc_kernel<<<nb(gs.numel()), 256, 0, n.s>>>(gscores, gs.p, f.N, hw, nc, A, a0);
      n.check_launch();
      out[i] = add(n, cv2[i].backward(n, gb), cv3[i].backward(n, gs));
      a0 += hw;
    }
  }
};

// ---------------------------------------------------------------------------------------------------------------
// the network: layer list with "up" / "cat" markers (Yolo.cs:53-89 / 209-257), outputs saved for the concats
// ---------------------------------------------------------------------------------------------------------------
struct Layer { int kind = 0; Mod m; };  // kind 0 module, 1 upsample, 2 concat

}  // namespace ts
}  // namespace yb

using namespace yb;
using namespace yb::ts;

struct yb_trainer {
  Net net;
  std::vector<Layer> layers;
  std::unique_ptr<Detect> detect;
  std::vector<int> output_idx;   // layers whose output is saved (Yolo.cs:13 / :202)
  int concat_index[4] = {1, 0, 3, 2};
  int feat_out[3] = {0, 0, 0};   // which saved outputs feed the head
  int A = 0;
  // per step
  std::vector<T4> outputs;
  std::vector<std::pair<int, int>> cat_split;  // (channels of the running tensor, saved output index) per concat
  std::vector<T4> up_in;
  float *boxes = nullptr, *scores = nullptr, *gboxes = nullptr, *gscores = nullptr, *items_dev = nullptr;
  int last_batch = 0;
  // targets of the step, staged before the forward pass is queued: host rows -> padded (B, n_max, 5) -> pinned -> device
  std::vector<float> tg_host;
  float* tg_pinned = nullptr;
  size_t tg_cap = 0;
  cudaEvent_t tg_copied = nullptr;
  // validation pass (yb_trainer_val_*): the accumulators live outside the arena, which every call resets.  Images and labels
  // are counted here; the detection row count and the loss sums only on the device (val.state / val.loss)
  bool val_on = false;
  ValAccum val{};
  void* val_block = nullptr;
  size_t val_bytes = 0;
  int val_max_images = 0, val_max_labels = 0, val_images = 0, val_labels = 0;
};

namespace {

const double V8_SZ[5][3] = {{0.34, 0.25, 1024}, {0.34, 0.5, 1024}, {0.67, 0.75, 576}, {1.0, 1.0, 512}, {1.0, 1.25, 640}};      // Yolo.cs:45-49
const double V11_SZ[5][4] = {{0.5, 0.25, 1024, 0}, {0.5, 0.5, 1024, 0}, {0.5, 1.0, 512, 1}, {1.0, 1.0, 512, 1}, {1.0, 1.5, 768, 1}};  // Yolo.cs:213-217

void add_mod(yb_trainer* t, Module* m) { Layer l; l.kind = 0; l.m.reset(m); t->layers.push_back(std::move(l)); }
void add_mark(yb_trainer* t, int kind) { Layer l; l.kind = kind; t->layers.push_back(std::move(l)); }

// every parameter / running statistic of a module tree is registered while the graph is built: the registry records the
// reference's state_dict names and shapes in construction order
struct Registry {
  std::vector<Entry> params, stats;
  void conv(const std::string& nm, int cin, int cout, int k, bool dw) {
    params.push_back({nm + ".conv.weight", {cout, dw ? 1 : cin, k, k}, 0, (long long)cout * (dw ? 1 : cin) * k * k, 0});
    params.push_back({nm + ".bn.weight", {cout}, 0, cout, 0});
    params.push_back({nm + ".bn.bias", {cout}, 0, cout, 0});
    stats.push_back({nm + ".bn.running_mean", {cout}, 0, cout, 1});
    stats.push_back({nm + ".bn.running_var", {cout}, 0, cout, 1});
  }
  void conv2d(const std::string& nm, int cin, int cout) {
    params.push_back({nm + ".weight", {cout, cin, 1, 1}, 0, (long long)cout * cin, 0});
    params.push_back({nm + ".bias", {cout}, 0, cout, 0});
  }
};

void reg_module(Registry& r, Module* m);
void reg_conv(Registry& r, Conv& c) { r.conv(c.name, c.cin, c.cout, c.k, c.depthwise != 0); }
void reg_module(Registry& r, Module* m) {
  if (auto* c = dynamic_cast<Conv*>(m)) { reg_conv(r, *c); return; }
  if (auto* c = dynamic_cast<Conv2dBias*>(m)) { r.conv2d(c->name, c->cin, c->cout); return; }
  if (auto* b = dynamic_cast<Bottleneck*>(m)) { reg_conv(r, b->cv1); reg_conv(r, b->cv2); return; }
  if (auto* c = dynamic_cast<C3k*>(m)) { reg_conv(r, c->cv1); reg_conv(r, c->cv2); reg_conv(r, c->cv3); for (auto& x : c->m) reg_module(r, x.get()); return; }
  if (auto* c = dynamic_cast<C2f*>(m)) { reg_conv(r, c->cv1); reg_conv(r, c->cv2); for (auto& x : c->m) reg_module(r, x.get()); return; }
  if (auto* s = dynamic_cast<SPPF*>(m)) { reg_conv(r, s->cv1); reg_conv(r, s->cv2); return; }
  if (auto* a = dynamic_cast<Attention*>(m)) { reg_conv(r, a->qkv); reg_conv(r, a->proj); reg_conv(r, a->pe); return; }
  if (auto* p = dynamic_cast<PSABlock*>(m)) { reg_module(r, &p->attn); reg_conv(r, p->f0); reg_conv(r, p->f1); return; }
  if (auto* c = dynamic_cast<C2PSA*>(m)) { reg_conv(r, c->cv1); reg_conv(r, c->cv2); for (auto& x : c->m) reg_module(r, x.get()); return; }
  if (auto* s = dynamic_cast<Seq*>(m)) { for (auto& x : s->layers) reg_module(r, x.get()); return; }
}

size_t max_workspace(yb_trainer* t);

int build(yb_trainer* t, int arch, int size, int nc) {
  Net& n = t->net;
  n.arch = arch; n.size = size; n.nc = nc;
  int w[5];
  if (arch == 8) {
    const double d = V8_SZ[size][0], wm = V8_SZ[size][1];
    const int mc = (int)V8_SZ[size][2];
    const int base[5] = {64, 128, 256, 512, 1024};
    for (int i = 0; i < 5; i++) w[i] = std::min((int)(base[i] * wm), mc);
    const int dp[3] = {(int)(3 * d), (int)(6 * d), (int)(9 * d)};
    // Yolo.cs:53-89
    add_mod(t, new Conv(n, "model.0", 3, w[0], 3, 2));
    add_mod(t, new Conv(n, "model.1", w[0], w[1], 3, 2));
    add_mod(t, new C2f(n, "model.2", w[1], w[1], dp[0], true, 0.5, 0));
    add_mod(t, new Conv(n, "model.3", w[1], w[2], 3, 2));
    add_mod(t, new C2f(n, "model.4", w[2], w[2], dp[1], true, 0.5, 0));
    add_mod(t, new Conv(n, "model.5", w[2], w[3], 3, 2));
    add_mod(t, new C2f(n, "model.6", w[3], w[3], dp[1], true, 0.5, 0));
    add_mod(t, new Conv(n, "model.7", w[3], w[4], 3, 2));
    add_mod(t, new C2f(n, "model.8", w[4], w[4], dp[0], true, 0.5, 0));
    add_mod(t, new SPPF(n, "model.9", w[4], w[4]));
    add_mark(t, 1); add_mark(t, 2);
    add_mod(t, new C2f(n, "model.12", w[4] + w[3], w[3], dp[0], false, 0.5, 0));
    add_mark(t, 1); add_mark(t, 2);
    add_mod(t, new C2f(n, "model.15", w[3] + w[2], w[2], dp[0], false, 0.5, 0));
    add_mod(t, new Conv(n, "model.16", w[2], w[2], 3, 2));
    add_mark(t, 2);
    add_mod(t, new C2f(n, "model.18", w[2] + w[3], w[3], dp[0], false, 0.5, 0));
    add_mod(t, new Conv(n, "model.19", w[3], w[3], 3, 2));
    add_mark(t, 2);
    add_mod(t, new C2f(n, "model.21", w[3] + w[4], w[4], dp[0], false, 0.5, 0));
    t->output_idx = {4, 6, 9, 12, 15, 18, 21};  // Yolo.cs:13
    const int ch[3] = {w[2], w[3], w[4]};
    t->detect.reset(new Detect(n, "model.22", nc, ch, true));
  } else if (arch == 11) {
    const double d = V11_SZ[size][0], wm = V11_SZ[size][1];
    const int mc = (int)V11_SZ[size][2];
    const bool c3k = V11_SZ[size][3] != 0;
    const int base[5] = {64, 128, 256, 512, 1024};
    for (int i = 0; i < 5; i++) w[i] = std::min((int)(base[i] * wm), mc);
    const int reps = (int)(2 * d);
    const int in_a = c3k ? 2 : 1;  // inner block of the C3k2 layers that follow the size's c3k flag
    // Yolo.cs:219-257
    add_mod(t, new Conv(n, "model.0", 3, w[0], 3, 2));
    add_mod(t, new Conv(n, "model.1", w[0], w[1], 3, 2));
    add_mod(t, new C2f(n, "model.2", w[1], w[2], reps, true, 0.25, in_a));
    add_mod(t, new Conv(n, "model.3", w[2], w[2], 3, 2));
    add_mod(t, new C2f(n, "model.4", w[2], w[3], reps, true, 0.25, in_a));
    add_mod(t, new Conv(n, "model.5", w[3], w[3], 3, 2));
    add_mod(t, new C2f(n, "model.6", w[3], w[3], reps, true, 0.5, 2));
    add_mod(t, new Conv(n, "model.7", w[3], w[4], 3, 2));
    add_mod(t, new C2f(n, "model.8", w[4], w[4], reps, true, 0.5, 2));
    add_mod(t, new SPPF(n, "model.9", w[4], w[4]));
    add_mod(t, new C2PSA(n, "model.10", w[4], reps));
    add_mark(t, 1); add_mark(t, 2);
    add_mod(t, new C2f(n, "model.13", w[4] + w[3], w[3], reps, true, 0.5, in_a));
    add_mark(t, 1); add_mark(t, 2);
    add_mod(t, new C2f(n, "model.16", w[3] + w[3], w[2], reps, true, 0.5, in_a));
    add_mod(t, new Conv(n, "model.17", w[2], w[2], 3, 2));
    add_mark(t, 2);
    add_mod(t, new C2f(n, "model.19", w[2] + w[3], w[3], reps, true, 0.5, in_a));
    add_mod(t, new Conv(n, "model.20", w[3], w[3], 3, 2));
    add_mark(t, 2);
    add_mod(t, new C2f(n, "model.22", w[3] + w[4], w[4], reps, true, 0.5, 2));
    t->output_idx = {4, 6, 10, 13, 16, 19, 22};  // Yolo.cs:202
    const int ch[3] = {w[2], w[3], w[4]};
    t->detect.reset(new Detect(n, "model.23", nc, ch, false));
  } else {
    set_error("yb_trainer_create: arch must be 8 or 11");
    return YB_ERR_INVALID_ARG;
  }
  auto* stem = dynamic_cast<Conv*>(t->layers[0].m.get());
  stem->pad8 = true;
  stem->need_dx = false;
  // registry -> flat layout: the reference's optimizer groups by name (YoloBaseTaskModel.cs:144-153): "bias" first
  Registry r;
  for (auto& l : t->layers) if (l.kind == 0) reg_module(r, l.m.get());
  for (int i = 0; i < 3; i++) { reg_module(r, &t->detect->cv2[i]); reg_module(r, &t->detect->cv3[i]); }
  std::vector<Entry> ordered;
  for (auto& e : r.params) if (e.name.find("bias") != std::string::npos) ordered.push_back(e);
  long long off = 0;
  for (auto& e : ordered) { e.off = off; off += e.count; }
  n.n_bias = off;
  for (auto& e : r.params) if (e.name.find("bias") == std::string::npos) { Entry c = e; c.off = off; off += c.count; ordered.push_back(c); }
  n.n_params = off;
  n.params = ordered;
  for (size_t i = 0; i < n.params.size(); i++) n.pidx[n.params[i].name] = (int)i;
  off = 0;
  for (auto& e : r.stats) { e.off = off; off += e.count; }
  n.n_stats = off;
  n.stats = r.stats;
  for (size_t i = 0; i < n.stats.size(); i++) n.sidx[n.stats[i].name] = (int)i;
  return YB_OK;
}

// workspace: the largest request of any dense conv at the planned batch / resolution (a dry walk over the shapes)
struct ShapeWalk {
  size_t ws = 0;
  int B;
  void conv(int H, int W, int cin, int cout, int k, int s) { ws = std::max(ws, tf_conv_workspace_bytes(B, H, W, cin, cout, k, s)); }
};
void walk_module(ShapeWalk& sw, Module* m, int& H, int& W) {
  if (auto* c = dynamic_cast<Conv*>(m)) {
    if (!c->depthwise) sw.conv(H, W, c->pad8 ? 8 : c->cin, c->cout, c->k, c->s);
    H = (H + 2 * (c->k / 2) - c->k) / c->s + 1; W = (W + 2 * (c->k / 2) - c->k) / c->s + 1;
    return;
  }
  if (auto* c = dynamic_cast<Conv2dBias*>(m)) { sw.conv(H, W, c->cin, c->cout, 1, 1); return; }
  int h = H, w = W;
  if (auto* b = dynamic_cast<Bottleneck*>(m)) { walk_module(sw, &b->cv1, h, w); walk_module(sw, &b->cv2, h, w); return; }
  if (auto* c = dynamic_cast<C3k*>(m)) { walk_module(sw, &c->cv1, h, w); walk_module(sw, &c->cv2, h, w); walk_module(sw, &c->cv3, h, w); for (auto& x : c->m) walk_module(sw, x.get(), h, w); return; }
  if (auto* c = dynamic_cast<C2f*>(m)) { walk_module(sw, &c->cv1, h, w); walk_module(sw, &c->cv2, h, w); for (auto& x : c->m) walk_module(sw, x.get(), h, w); return; }
  if (auto* s = dynamic_cast<SPPF*>(m)) { walk_module(sw, &s->cv1, h, w); walk_module(sw, &s->cv2, h, w); return; }
  if (auto* a = dynamic_cast<Attention*>(m)) { walk_module(sw, &a->qkv, h, w); walk_module(sw, &a->proj, h, w); return; }
  if (auto* p = dynamic_cast<PSABlock*>(m)) { walk_module(sw, &p->attn, h, w); walk_module(sw, &p->f0, h, w); walk_module(sw, &p->f1, h, w); return; }
  if (auto* c = dynamic_cast<C2PSA*>(m)) { walk_module(sw, &c->cv1, h, w); walk_module(sw, &c->cv2, h, w); for (auto& x : c->m) walk_module(sw, x.get(), h, w); return; }
  if (auto* s = dynamic_cast<Seq*>(m)) { for (auto& x : s->layers) walk_module(sw, x.get(), h, w); return; }
}
size_t max_workspace(yb_trainer* t) {
  ShapeWalk sw;
  sw.B = t->net.max_batch;
  int H = t->net.H, W = t->net.W;
  std::vector<std::pair<int, int>> saved;
  for (size_t i = 0; i < t->layers.size(); i++) {
    Layer& l = t->layers[i];
    if (l.kind == 1) { H *= 2; W *= 2; }
    else if (l.kind == 0) walk_module(sw, l.m.get(), H, W);
    // concat keeps the spatial size of the running tensor
  }
  const int strides[3] = {8, 16, 32};
  for (int i = 0; i < 3; i++) {
    int h = t->net.H / strides[i], w = t->net.W / strides[i];
    walk_module(sw, &t->detect->cv2[i], h, w);
    h = t->net.H / strides[i]; w = t->net.W / strides[i];
    walk_module(sw, &t->detect->cv3[i], h, w);
  }
  return sw.ws + 4096;
}

// the layer walk of Yolo.cs:92-134 up to the Detect head, in train or eval mode (n.eval): saves the outputs the concats and
// the backward pass read, returns the three head inputs
int forward_layers(yb_trainer* t, T4 x, T4 feats[3]) {
  Net& n = t->net;
  t->outputs.clear();
  t->cat_split.clear();
  t->up_in.clear();
  int cat_count = 0;
  for (size_t i = 0; i < t->layers.size() && !n.rc; i++) {
    Layer& l = t->layers[i];
    if (l.kind == 1) {
      T4 y = n.make(x.N, 2 * x.H, 2 * x.W, x.C);
      if (n.rc) break;
      up2_forward_kernel<<<nb(y.numel()), 256, 0, n.s>>>(x.p, x.pitch, y.p, y.pitch, x.N, x.H, x.W, x.C);
      n.check_launch();
      t->up_in.push_back(x);
      x = y;
    } else if (l.kind == 2) {
      const T4& other = t->outputs[t->concat_index[cat_count]];
      t->cat_split.push_back({x.C, t->concat_index[cat_count]});
      T4 y = n.make(x.N, x.H, x.W, x.C + other.C);
      put(n, y, 0, x);
      put(n, y, x.C, other);
      x = y;
      cat_count++;
    } else {
      x = l.m->forward(n, x);
    }
    if (std::find(t->output_idx.begin(), t->output_idx.end(), (int)i) != t->output_idx.end()) t->outputs.push_back(x);
  }
  if (n.rc) return n.rc;
  const int n_out = (int)t->outputs.size();
  for (int k = 0; k < 3; k++) feats[k] = t->outputs[n_out - 3 + k];
  return YB_OK;
}

// t->tg_host -> the pinned staging buffer -> the arena, queued on s.  The pinned buffer is reused by the next call: it is
// only overwritten once the copy queued by the previous call has left it (tg_copied), the one host wait of a call.
int stage_targets(yb_trainer* t, cudaStream_t s, const char* who, float** d_out) {
  Net& n = t->net;
  const std::string w(who);
  if (!t->tg_copied && cudaEventCreateWithFlags(&t->tg_copied, cudaEventDisableTiming) != cudaSuccess) { set_error(w + ": cudaEventCreate failed"); return YB_ERR_CUDA; }
  if (t->tg_pinned && cudaEventSynchronize(t->tg_copied) != cudaSuccess) { set_error(w + ": cudaEventSynchronize failed"); return YB_ERR_CUDA; }
  if (t->tg_host.size() > t->tg_cap) {
    if (t->tg_pinned) cudaFreeHost(t->tg_pinned);
    t->tg_pinned = nullptr;
    t->tg_cap = std::max<size_t>(t->tg_host.size() * 2, 4096);
    if (cudaMallocHost((void**)&t->tg_pinned, t->tg_cap * sizeof(float)) != cudaSuccess) { t->tg_cap = 0; set_error(w + ": cudaMallocHost failed"); return YB_ERR_CUDA; }
  }
  memcpy(t->tg_pinned, t->tg_host.data(), t->tg_host.size() * sizeof(float));
  float* d = n.alloc((long long)t->tg_host.size());
  if (n.rc) return n.rc;
  if (cudaMemcpyAsync(d, t->tg_pinned, t->tg_host.size() * sizeof(float), cudaMemcpyHostToDevice, s) != cudaSuccess ||
      cudaEventRecord(t->tg_copied, s) != cudaSuccess) { set_error(w + ": target copy failed"); return YB_ERR_CUDA; }
  *d_out = d;
  return YB_OK;
}

// forward + loss + backward of one batch; gradients land in the caller's flat buffer
int run_backward(yb_trainer* t, const void* images, int in_dtype, int B, const float* targets_host, int n_targets, float* items_host,
                 cudaStream_t s) {
  Net& n = t->net;
  n.s = s;
  n.rc = 0;
  n.arena_off = 0;
  const int H = n.H, W = n.W;
  T4 x = n.make(B, H, W, 8);
  if (n.rc) return n.rc;
  // targets first: the host never waits on the stream between here and the end of the backward pass, so the launches of the
  // whole step queue up behind the running kernels (the loss used to synchronise to hand over a host temporary: the
  // backward pass then started from an empty queue)
  int n_max = 0;
  if (int rc = detection_loss_prepare(targets_host, n_targets, B, n.nc, H, W, t->tg_host, &n_max)) return rc;
  float* d_gts = nullptr;
  if (int rc = stage_targets(t, s, "yb_train_step", &d_gts)) return rc;
  images_to_nhwc8_kernel<<<nb((long long)B * H * W), 256, 0, s>>>(images, in_dtype == YB_U8 ? 1 : 0, x.p, B, H, W);
  n.check_launch();
  n.check(tf_pack_all(n.P, n.WF, n.WB, n.pack_descs, n.n_packs, n.pack_chunks, s));  // the weights as this step sees them
  T4 feats[3];
  if (int rc = forward_layers(t, x, feats)) return rc;
  const int n_out = (int)t->outputs.size();
  const int A = feats[0].H * feats[0].W + feats[1].H * feats[1].W + feats[2].H * feats[2].W;
  t->A = A;
  t->boxes = n.alloc((long long)B * 64 * A);
  t->scores = n.alloc((long long)B * n.nc * A);
  t->gboxes = n.alloc((long long)B * 64 * A);
  t->gscores = n.alloc((long long)B * n.nc * A);
  t->items_dev = n.alloc(4);
  unsigned char* fg = reinterpret_cast<unsigned char*>(n.alloc(((long long)B * A + 3) / 4 + 1));
  int* gt_idx = reinterpret_cast<int*>(n.alloc((long long)B * A));
  float* tsc = n.alloc((long long)B * A);
  if (n.rc) return n.rc;
  t->detect->forward(n, feats, t->boxes, t->scores, A);
  if (n.rc) return n.rc;
  // ---- loss (Loss.cs:328-485) and its gradient w.r.t. the head outputs ----
  n.check(detection_loss_launch_dev(t->boxes, t->scores, B, n.nc, 16, H, W, d_gts, n_max, 10, 7.5f, 0.5f, 1.5f, t->items_dev,
                                    t->gboxes, t->gscores, fg, gt_idx, tsc, s));
  if (n.rc) return n.rc;
  // ---- backward through the graph ----
  if (cudaMemsetAsync(n.G, 0, (size_t)n.n_params * sizeof(float), s) != cudaSuccess) { set_error("yb_train_step: memset failed"); return YB_ERR_CUDA; }
  T4 dfeat[3];
  t->detect->backward(n, t->gboxes, t->gscores, A, dfeat);
  if (n.rc) return n.rc;
  std::vector<T4> dout(n_out);
  std::vector<char> has(n_out, 0);
  for (int k = 0; k < 3; k++) { dout[n_out - 3 + k] = dfeat[k]; has[n_out - 3 + k] = 1; }
  T4 dx;
  bool have_dx = false;
  int cc = (int)t->cat_split.size(), up = (int)t->up_in.size();
  for (int i = (int)t->layers.size() - 1; i >= 0 && !n.rc; i--) {
    auto it = std::find(t->output_idx.begin(), t->output_idx.end(), i);
    if (it != t->output_idx.end()) {
      const int j = (int)(it - t->output_idx.begin());
      if (has[j]) {
        dx = have_dx ? add(n, dx, dout[j]) : dout[j];
        have_dx = true;
      }
    }
    Layer& l = t->layers[i];
    if (l.kind == 1) {
      up--;
      const T4& xin = t->up_in[up];
      T4 d = n.make(xin.N, xin.H, xin.W, xin.C);
      if (n.rc) break;
      up2_backward_kernel<<<nb(d.numel()), 256, 0, s>>>(dx.p, dx.pitch, d.p, xin.N, xin.H, xin.W, xin.C);
      n.check_launch();
      dx = d;
    } else if (l.kind == 2) {
      cc--;
      const int cx = t->cat_split[cc].first, src = t->cat_split[cc].second;
      const T4 d_other = view(dx, cx, dx.C - cx);  // views of the concat's gradient: no copies
      dout[src] = has[src] ? add(n, dout[src], d_other) : d_other;
      has[src] = 1;
      dx = view(dx, 0, cx);
    } else {
      dx = l.m->backward(n, dx);
    }
  }
  if (n.rc) return n.rc;
  if (items_host) {
    if (cudaMemcpyAsync(items_host, t->items_dev, 3 * sizeof(float), cudaMemcpyDeviceToHost, s) != cudaSuccess ||
        cudaStreamSynchronize(s) != cudaSuccess) {
      set_error(std::string("yb_train_step: ") + cudaGetErrorString(cudaGetLastError()));
      return YB_ERR_CUDA;
    }
  }
  t->last_batch = B;
  return YB_OK;
}

// eval mode: the fold descriptors of every conv (pointers into the bound buffers and EV), built on first use after a bind
int prepare_eval(yb_trainer* t) {
  Net& n = t->net;
  if (n.fold_descs) return YB_OK;
  if (!n.EV && cudaMalloc((void**)&n.EV, (size_t)n.n_params * sizeof(float)) != cudaSuccess) {
    n.EV = nullptr;
    cudaGetLastError();
    set_error("yb_trainer_evaluate: cudaMalloc of the folded weight buffer failed");
    return YB_ERR_CUDA;
  }
  std::vector<TfFoldDesc> d;
  long long chunk = 0;
  const std::string cw = ".conv.weight";
  for (auto& e : n.params) {
    if (e.shape.size() != 4) continue;
    TfFoldDesc q{};
    q.w = n.P + e.off;
    q.cout = (int)e.shape[0]; q.cin = (int)e.shape[1]; q.taps = (int)(e.shape[2] * e.shape[3]);
    const bool dense = q.cout % 8 == 0 && q.cin % 8 == 0;  // the stem (3 channels) and depthwise convs keep their own kernels
    if (e.name.size() > cw.size() && e.name.compare(e.name.size() - cw.size(), cw.size(), cw) == 0) {
      const std::string b = e.name.substr(0, e.name.size() - cw.size());
      q.gamma = n.p(b + ".bn.weight"); q.beta = n.p(b + ".bn.bias");
      q.rm = n.r(b + ".bn.running_mean"); q.rv = n.r(b + ".bn.running_var");
      q.bias = n.ev(b + ".bn.bias"); q.invstd = n.ev(b + ".bn.weight");
    } else if (!dense) {
      continue;  // a plain Conv2d the eval forward does not run on the tensor cores (none in the detect graphs)
    }
    q.wf = dense ? n.EV + e.off : nullptr;
    q.chunk0 = chunk;
    chunk += tf_fold_chunks(q);
    d.push_back(q);
  }
  if (cudaMalloc((void**)&n.fold_descs, std::max<size_t>(1, d.size()) * sizeof(TfFoldDesc)) != cudaSuccess ||
      cudaMemcpy(n.fold_descs, d.data(), d.size() * sizeof(TfFoldDesc), cudaMemcpyHostToDevice) != cudaSuccess) {
    if (n.fold_descs) cudaFree(n.fold_descs);
    n.fold_descs = nullptr;
    cudaGetLastError();
    set_error("yb_trainer_evaluate: fold descriptor upload failed");
    return YB_ERR_CUDA;
  }
  n.n_folds = (int)d.size();
  n.fold_chunks = chunk;
  return YB_OK;
}

int anchors(const Net& n) { return (n.H / 8) * (n.W / 8) + (n.H / 16) * (n.W / 16) + (n.H / 32) * (n.W / 32); }

// the eval-mode forward (`AMPWrapper.Evaluate`) on the arena as the caller left it: one fold launch, then the layer walk
// and the head with BatchNorm folded; pred / boxes / scores each optional
int eval_forward(yb_trainer* t, const void* images, int in_dtype, int B, float* pred, float* boxes, float* scores) {
  if (int rc = prepare_eval(t)) return rc;
  Net& n = t->net;
  T4 x = n.make(B, n.H, n.W, 8);
  if (n.rc) return n.rc;
  images_to_nhwc8_kernel<<<nb((long long)B * n.H * n.W), 256, 0, n.s>>>(images, in_dtype == YB_U8 ? 1 : 0, x.p, B, n.H, n.W);
  n.check_launch();
  n.check(tf_fold_all(n.fold_descs, n.n_folds, n.fold_chunks, n.s));  // BatchNorm as the current parameters and statistics give it
  n.eval = true;
  T4 feats[3];
  int rc = forward_layers(t, x, feats);
  if (!rc) {
    t->detect->forward(n, feats, boxes, scores, anchors(n), pred);
    rc = n.rc;
  }
  n.eval = false;
  return rc;
}

}  // namespace

extern "C" {

int32_t yb_trainer_create(const yb_config* cfg, yb_trainer** out) {
  if (!cfg || !out) { set_error("yb_trainer_create: null argument"); return YB_ERR_INVALID_ARG; }
  if (cfg->task != YB_TASK_DETECT) { set_error("yb_trainer_create: detect models only"); return YB_ERR_NOT_IMPLEMENTED; }
  if (cfg->size < 0 || cfg->size > 4 || cfg->nc <= 0 || cfg->max_batch <= 0 || cfg->height <= 0 || cfg->width <= 0 || cfg->height % 32 ||
      cfg->width % 32) {
    set_error("yb_trainer_create: size in 0..4, nc > 0, max_batch > 0, height / width multiples of 32");
    return YB_ERR_INVALID_ARG;
  }
  std::unique_ptr<yb_trainer> t(new yb_trainer());
  t->net.max_batch = cfg->max_batch;
  t->net.H = cfg->height;
  t->net.W = cfg->width;
  if (int rc = build(t.get(), cfg->arch, cfg->size, cfg->nc)) return rc;
  if (cfg->flags & YB_FLAG_DRY_RUN) { *out = t.release(); return YB_OK; }  // names / layout only (CPU tests)
  if (!have_device("yb_trainer_create")) return YB_ERR_NO_DEVICE;
  if (cudaSetDevice(cfg->device) != cudaSuccess) { set_error("yb_trainer_create: cudaSetDevice failed"); cudaGetLastError(); return YB_ERR_CUDA; }
  {
    // the kernels' scratch (BatchNorm partials, attention statistics, ...) comes from the stream-ordered allocator; by
    // default its pool hands unused memory back to the OS at every synchronisation - and a step ends with one (loss items
    // to the host) - so the next step would pay for fresh device allocations (random slow steps)
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, cfg->device) == cudaSuccess) {
      uint64_t keep = UINT64_MAX;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    }
    cudaGetLastError();
  }
  t->net.ws_bytes = max_workspace(t.get());
  // activations + gradients of one step: every conv block keeps x, z, y (+ dz, dx on the way back); sized from the fp32
  // activation volume of the model at this batch with headroom, grown on demand is not possible inside a step
  const double act_mb_per_img = (t->net.arch == 11 ? 1500.0 : 1100.0) * (t->net.size >= 2 ? 3.0 : (t->net.size == 1 ? 1.6 : 1.0)) *
                                ((double)cfg->height * cfg->width / (640.0 * 640.0));
  t->net.arena_cap = (size_t)(act_mb_per_img * 1e6 * cfg->max_batch) + ((size_t)256 << 20);
  if (cudaMalloc((void**)&t->net.ws, t->net.ws_bytes) != cudaSuccess || cudaMalloc((void**)&t->net.arena, t->net.arena_cap) != cudaSuccess) {
    set_error("yb_trainer_create: cudaMalloc of the workspace / activation arena failed");
    cudaGetLastError();
    if (t->net.ws) cudaFree(t->net.ws);
    return YB_ERR_CUDA;
  }
  {
    // tensor-core operand copies of every dense conv weight (forward [tap][Cout][Cin], dgrad [tap][Cin][Cout]) at the
    // offsets of the checkpoint-layout tensors; one pack launch per step
    Net& n = t->net;
    std::vector<TfPackDesc> d;
    long long chunk = 0;
    for (auto& e : n.params) {
      if (e.shape.size() != 4 || e.shape[0] % 8 || e.shape[1] % 8 || e.shape[2] != e.shape[3] || (e.shape[2] != 1 && e.shape[2] != 3)) continue;
      TfPackDesc q{};
      q.off = e.off; q.chunk0 = chunk; q.cout = (int)e.shape[0]; q.cin = (int)e.shape[1]; q.taps = (int)(e.shape[2] * e.shape[3]);
      chunk += tf_pack_chunks(q.cout, q.cin, q.taps);
      d.push_back(q);
    }
    n.n_packs = (int)d.size();
    n.pack_chunks = chunk;
    const size_t wbytes = (size_t)n.n_params * sizeof(float);
    if (cudaMalloc((void**)&n.WF, wbytes) != cudaSuccess || cudaMalloc((void**)&n.WB, wbytes) != cudaSuccess ||
        cudaMalloc((void**)&n.pack_descs, std::max<size_t>(1, d.size()) * sizeof(TfPackDesc)) != cudaSuccess ||
        cudaMalloc((void**)&n.bn_counters, 64 * sizeof(unsigned)) != cudaSuccess || cudaMemset(n.bn_counters, 0, 64 * sizeof(unsigned)) != cudaSuccess ||
        cudaMemcpy(n.pack_descs, d.data(), d.size() * sizeof(TfPackDesc), cudaMemcpyHostToDevice) != cudaSuccess) {
      set_error("yb_trainer_create: cudaMalloc of the packed weight buffers failed");
      cudaGetLastError();
      yb_trainer_destroy(t.release());
      return YB_ERR_CUDA;
    }
  }
  *out = t.release();
  return YB_OK;
}

void yb_trainer_destroy(yb_trainer* t) {
  if (!t) return;
  if (t->net.ws) cudaFree(t->net.ws);
  if (t->net.arena) cudaFree(t->net.arena);
  if (t->net.WF) cudaFree(t->net.WF);
  if (t->net.WB) cudaFree(t->net.WB);
  if (t->net.pack_descs) cudaFree(t->net.pack_descs);
  if (t->net.bn_counters) cudaFree(t->net.bn_counters);
  if (t->net.EV) cudaFree(t->net.EV);
  if (t->net.fold_descs) cudaFree(t->net.fold_descs);
  if (t->tg_pinned) cudaFreeHost(t->tg_pinned);
  if (t->tg_copied) cudaEventDestroy(t->tg_copied);
  if (t->val_block) cudaFree(t->val_block);
  delete t;
}

int32_t yb_trainer_num_tensors(const yb_trainer* t, int32_t kind) {
  if (!t) return 0;
  return (int32_t)(kind == 0 ? t->net.params.size() : t->net.stats.size());
}

int32_t yb_trainer_tensor_info(const yb_trainer* t, int32_t kind, int32_t index, const char** name, int64_t* offset, int64_t* count,
                               int32_t* ndim, const int64_t** shape) {
  if (!t) { set_error("yb_trainer_tensor_info: null trainer"); return YB_ERR_INVALID_ARG; }
  const std::vector<Entry>& v = kind == 0 ? t->net.params : t->net.stats;
  if (index < 0 || index >= (int)v.size()) { set_error("yb_trainer_tensor_info: index out of range"); return YB_ERR_INVALID_ARG; }
  const Entry& e = v[index];
  if (name) *name = e.name.c_str();
  if (offset) *offset = e.off;
  if (count) *count = e.count;
  if (ndim) *ndim = (int32_t)e.shape.size();
  if (shape) *shape = e.shape.data();
  return YB_OK;
}

int64_t yb_trainer_flat_size(const yb_trainer* t, int32_t kind) {
  if (!t) return 0;
  return kind == 0 ? t->net.n_params : (kind == 1 ? t->net.n_stats : t->net.n_bias);
}

int32_t yb_trainer_bind(yb_trainer* t, float* params, float* grads, float* adam_m, float* adam_v, float* running_stats) {
  if (!t || !params || !grads || !adam_m || !adam_v || !running_stats) { set_error("yb_trainer_bind: null argument"); return YB_ERR_INVALID_ARG; }
  t->net.P = params; t->net.G = grads; t->net.M1 = adam_m; t->net.M2 = adam_v; t->net.R = running_stats;
  if (t->net.fold_descs) { cudaFree(t->net.fold_descs); t->net.fold_descs = nullptr; }  // they point into the old buffers
  return YB_OK;
}

int32_t yb_train_backward(yb_trainer* t, const void* images, int32_t in_dtype, int32_t batch, const float* targets_host,
                          int32_t n_targets, float* loss_items_host, void* stream) {
  if (!t || !images) { set_error("yb_train_backward: null argument"); return YB_ERR_INVALID_ARG; }
  if (!t->net.P || !t->net.arena) { set_error("yb_train_backward: call yb_trainer_bind first (and create without DRY_RUN)"); return YB_ERR_STATE; }
  if (batch <= 0 || batch > t->net.max_batch) { set_error("yb_train_backward: batch outside [1, max_batch]"); return YB_ERR_INVALID_ARG; }
  if (in_dtype != YB_U8 && in_dtype != YB_F32) { set_error("yb_train_backward: images must be u8 or f32 NCHW"); return YB_ERR_INVALID_ARG; }
  if (n_targets < 0 || (n_targets > 0 && !targets_host)) { set_error("yb_train_backward: bad targets"); return YB_ERR_INVALID_ARG; }
  return run_backward(t, images, in_dtype, batch, targets_host, n_targets, loss_items_host, (cudaStream_t)stream);
}

int32_t yb_train_apply(yb_trainer* t, float lr_bias, float lr_other, float weight_decay, void* stream) {
  if (!t || !t->net.P) { set_error("yb_train_apply: trainer not bound"); return YB_ERR_STATE; }
  Net& n = t->net;
  n.step_count++;
  cudaStream_t s = (cudaStream_t)stream;
  // AdamW(lr, weight_decay 5e-4, betas 0.9 / 0.999, eps 1e-8) per name group (YoloBaseTaskModel.cs:142-160)
  if (n.n_bias > 0)
    if (int rc = adamw_step(n.P, n.G, n.M1, n.M2, n.n_bias, n.step_count, lr_bias, 0.9f, 0.999f, 1e-8f, weight_decay, s)) return rc;
  if (n.n_params > n.n_bias)
    if (int rc = adamw_step(n.P + n.n_bias, n.G + n.n_bias, n.M1 + n.n_bias, n.M2 + n.n_bias, n.n_params - n.n_bias, n.step_count, lr_other, 0.9f,
                            0.999f, 1e-8f, weight_decay, s))
      return rc;
  return YB_OK;
}

int32_t yb_train_step(yb_trainer* t, const void* images, int32_t in_dtype, int32_t batch, const float* targets_host, int32_t n_targets,
                      float lr_bias, float lr_other, float weight_decay, float* loss_items_host, void* stream) {
  if (int rc = yb_train_backward(t, images, in_dtype, batch, targets_host, n_targets, loss_items_host, stream)) return rc;
  return yb_train_apply(t, lr_bias, lr_other, weight_decay, stream);
}

int32_t yb_trainer_evaluate(yb_trainer* t, const void* images, int32_t in_dtype, int32_t batch, float* pred, float* boxes,
                            float* scores, void* stream) {
  if (!t || !images) { set_error("yb_trainer_evaluate: null argument"); return YB_ERR_INVALID_ARG; }
  if (!t->net.P || !t->net.arena) { set_error("yb_trainer_evaluate: call yb_trainer_bind first (and create without DRY_RUN)"); return YB_ERR_STATE; }
  if (batch <= 0 || batch > t->net.max_batch) { set_error("yb_trainer_evaluate: batch outside [1, max_batch]"); return YB_ERR_INVALID_ARG; }
  if (in_dtype != YB_U8 && in_dtype != YB_F32) { set_error("yb_trainer_evaluate: images must be u8 or f32 NCHW"); return YB_ERR_INVALID_ARG; }
  if (!have_device("yb_trainer_evaluate")) return YB_ERR_NO_DEVICE;
  Net& n = t->net;
  n.s = (cudaStream_t)stream;
  n.rc = 0;
  n.arena_off = 0;
  return eval_forward(t, images, in_dtype, batch, pred, boxes, scores);
}

int32_t yb_trainer_val_begin(yb_trainer* t, int32_t max_images, int32_t max_labels, void* stream) {
  if (!t) { set_error("yb_trainer_val_begin: null trainer"); return YB_ERR_INVALID_ARG; }
  if (!t->net.P || !t->net.arena) { set_error("yb_trainer_val_begin: call yb_trainer_bind first (and create without DRY_RUN)"); return YB_ERR_STATE; }
  if (max_images <= 0 || max_labels <= 0 || (long long)max_images * VAL_MAX_DET > INT32_MAX) {
    set_error("yb_trainer_val_begin: need max_images > 0 (at most 2^31 / 300) and max_labels > 0");
    return YB_ERR_INVALID_ARG;
  }
  if (!have_device("yb_trainer_val_begin")) return YB_ERR_NO_DEVICE;
  cudaStream_t s = (cudaStream_t)stream;
  const size_t rows = (size_t)max_images * VAL_MAX_DET;
  auto up = [](size_t b) { return (b + 255) & ~(size_t)255; };
  const size_t o_conf = up(rows * VAL_T), o_cls = o_conf + up(rows * 4), o_tcls = o_cls + up(rows * 4),
               o_state = o_tcls + up((size_t)max_labels * 4), bytes = o_state + 256;
  t->val_on = false;
  if (bytes > t->val_bytes) {
    if (t->val_block) cudaFree(t->val_block);
    t->val_block = nullptr;
    t->val_bytes = 0;
    if (cudaMalloc(&t->val_block, bytes) != cudaSuccess) {
      t->val_block = nullptr;
      cudaGetLastError();
      set_error("yb_trainer_val_begin: cudaMalloc of the validation accumulators failed");
      return YB_ERR_CUDA;
    }
    t->val_bytes = bytes;
  }
  char* b = static_cast<char*>(t->val_block);
  ValAccum& a = t->val;
  a.tp = reinterpret_cast<unsigned char*>(b);
  a.conf = reinterpret_cast<float*>(b + o_conf);
  a.cls = reinterpret_cast<int*>(b + o_cls);
  a.target_cls = reinterpret_cast<int*>(b + o_tcls);
  a.state = reinterpret_cast<int*>(b + o_state);
  a.loss = reinterpret_cast<float*>(b + o_state + 16);
  a.cap_rows = (long long)rows;
  YB_CUDA_CHECK(cudaMemsetAsync(a.state, 0, 256, s));  // row count, overflow flag, loss sums
  t->val_max_images = max_images;
  t->val_max_labels = max_labels;
  t->val_images = t->val_labels = 0;
  t->val_on = true;
  return YB_OK;
}

int32_t yb_trainer_val_batch(yb_trainer* t, const void* images, int32_t in_dtype, int32_t batch, const float* targets_host,
                             int32_t n_targets, void* stream) {
  if (!t || !images) { set_error("yb_trainer_val_batch: null argument"); return YB_ERR_INVALID_ARG; }
  if (!t->val_on) { set_error("yb_trainer_val_batch: call yb_trainer_val_begin first"); return YB_ERR_STATE; }
  if (batch <= 0 || batch > t->net.max_batch) { set_error("yb_trainer_val_batch: batch outside [1, max_batch]"); return YB_ERR_INVALID_ARG; }
  if (in_dtype != YB_U8 && in_dtype != YB_F32) { set_error("yb_trainer_val_batch: images must be u8 or f32 NCHW"); return YB_ERR_INVALID_ARG; }
  if (n_targets < 0 || (n_targets > 0 && !targets_host)) { set_error("yb_trainer_val_batch: bad targets"); return YB_ERR_INVALID_ARG; }
  if (n_targets == 0) return YB_OK;  // Detector.cs:91-94: a batch without labels is skipped - no loss, rows or image count
  if (t->val_images + batch > t->val_max_images || t->val_labels + n_targets > t->val_max_labels) {
    set_error("yb_trainer_val_batch: more images or labels than yb_trainer_val_begin was sized for");
    return YB_ERR_INVALID_ARG;
  }
  if (n_targets > VAL_MAX_BATCH_LABELS) { set_error("yb_trainer_val_batch: at most 2048 labels per batch"); return YB_ERR_INVALID_ARG; }
  Net& n = t->net;
  const int B = batch, H = n.H, W = n.W;
  int n_max = 0;
  // the loss's padded (B, n_max, 5) targets; validates image indices and class ids
  if (int rc = detection_loss_prepare(targets_host, n_targets, B, n.nc, H, W, t->tg_host, &n_max)) return rc;
  // followed by the raw rows, stably sorted by image: the order in which Detector.Val concatenates each image's labels
  const size_t gts = t->tg_host.size();
  std::vector<int> start(B + 1, 0);
  for (int i = 0; i < n_targets; i++) start[(int)targets_host[(size_t)i * 6] + 1]++;
  for (int b = 0; b < B; b++) start[b + 1] += start[b];
  t->tg_host.resize(gts + (size_t)n_targets * 6);
  for (int i = 0; i < n_targets; i++) {
    const float* r = targets_host + (size_t)i * 6;
    std::copy(r, r + 6, t->tg_host.begin() + gts + (size_t)start[(int)r[0]]++ * 6);
  }
  n.s = (cudaStream_t)stream;
  n.rc = 0;
  n.arena_off = 0;
  float* d_tg = nullptr;
  if (int rc = stage_targets(t, n.s, "yb_trainer_val_batch", &d_tg)) return rc;
  const int A = anchors(n);
  float* pred = n.alloc((long long)B * (4 + n.nc) * A);
  float* boxes = n.alloc((long long)B * 64 * A);
  float* scores = n.alloc((long long)B * n.nc * A);
  float* items = n.alloc(4);
  float* labels = n.alloc((long long)n_targets * 6);
  float* dets = n.alloc((long long)B * VAL_MAX_DET * 6);
  int* counts = reinterpret_cast<int*>(n.alloc(B));
  unsigned char* correct = reinterpret_cast<unsigned char*>(n.alloc(((long long)B * VAL_MAX_DET * VAL_T + 3) / 4));
  if (n.rc) return n.rc;
  if (int rc = eval_forward(t, images, in_dtype, B, pred, boxes, scores)) return rc;
  // v8DetectionLoss without gradients: `loss.forward(preds, data).loss_detach` (Detector.cs:96)
  if (int rc = detection_loss_launch_dev(boxes, scores, B, n.nc, 16, H, W, d_tg, n_max, 10, 7.5f, 0.5f, 1.5f, items, nullptr, nullptr,
                                         nullptr, nullptr, nullptr, n.s))
    return rc;
  if (int rc = val_batch_launch(pred, B, n.nc, A, H, W, d_tg + gts, n_targets, t->val_labels, items, labels, dets, counts, correct, t->val,
                                n.s))
    return rc;
  t->val_images += B;
  t->val_labels += n_targets;
  return YB_OK;
}

int32_t yb_trainer_val_append(yb_trainer* t, const uint8_t* tp, const float* conf, const int32_t* pred_cls, int32_t n,
                              const int32_t* target_cls, int32_t m, void* stream) {
  if (!t) { set_error("yb_trainer_val_append: null trainer"); return YB_ERR_INVALID_ARG; }
  if (!t->val_on) { set_error("yb_trainer_val_append: call yb_trainer_val_begin first"); return YB_ERR_STATE; }
  if (n < 0 || m < 0 || (n > 0 && (!tp || !conf || !pred_cls)) || (m > 0 && !target_cls)) { set_error("yb_trainer_val_append: bad argument"); return YB_ERR_INVALID_ARG; }
  if (t->val_labels + m > t->val_max_labels) { set_error("yb_trainer_val_append: more labels than yb_trainer_val_begin was sized for"); return YB_ERR_INVALID_ARG; }
  if (n == 0 && m == 0) return YB_OK;
  if (int rc = val_append_launch(tp, conf, pred_cls, n, target_cls, m, t->val_labels, t->val, (cudaStream_t)stream)) return rc;
  t->val_labels += m;
  return YB_OK;
}

int32_t yb_trainer_val_rows(yb_trainer* t, uint8_t* tp, float* conf, int32_t* pred_cls, int32_t* target_cls, int32_t* counts_host,
                            int32_t clear, void* stream) {
  if (!t || !counts_host) { set_error("yb_trainer_val_rows: null argument"); return YB_ERR_INVALID_ARG; }
  if (!t->val_on) { set_error("yb_trainer_val_rows: call yb_trainer_val_begin first"); return YB_ERR_STATE; }
  cudaStream_t s = (cudaStream_t)stream;
  int st[2] = {0, 0};
  YB_CUDA_CHECK(cudaMemcpyAsync(st, t->val.state, sizeof(st), cudaMemcpyDeviceToHost, s));
  YB_CUDA_CHECK(cudaStreamSynchronize(s));
  if (st[1]) { set_error("yb_trainer_val_rows: the detection rows overflowed the accumulators"); return YB_ERR_STATE; }
  const int n = st[0], m = t->val_labels;
  counts_host[0] = n;
  counts_host[1] = m;
  if (tp && n) YB_CUDA_CHECK(cudaMemcpyAsync(tp, t->val.tp, (size_t)n * VAL_T, cudaMemcpyDeviceToDevice, s));
  if (conf && n) YB_CUDA_CHECK(cudaMemcpyAsync(conf, t->val.conf, (size_t)n * 4, cudaMemcpyDeviceToDevice, s));
  if (pred_cls && n) YB_CUDA_CHECK(cudaMemcpyAsync(pred_cls, t->val.cls, (size_t)n * 4, cudaMemcpyDeviceToDevice, s));
  if (target_cls && m) YB_CUDA_CHECK(cudaMemcpyAsync(target_cls, t->val.target_cls, (size_t)m * 4, cudaMemcpyDeviceToDevice, s));
  if (clear) {
    YB_CUDA_CHECK(cudaMemsetAsync(t->val.state, 0, sizeof(int), s));  // the row count; loss sums and the image count stay
    t->val_labels = 0;
  }
  return YB_OK;
}

int32_t yb_trainer_val_end(yb_trainer* t, float* loss_items_host, float* metrics_host, int32_t* counts_host, void* stream) {
  if (!t || !loss_items_host || !metrics_host || !counts_host) { set_error("yb_trainer_val_end: null argument"); return YB_ERR_INVALID_ARG; }
  if (!t->val_on) { set_error("yb_trainer_val_end: call yb_trainer_val_begin first"); return YB_ERR_STATE; }
  // every executed batch has labels, so no labels means nothing was accumulated (the reference's torch.cat of empty lists throws)
  if (t->val_labels == 0) { set_error("yb_trainer_val_end: no batch with labels was validated"); return YB_ERR_STATE; }
  cudaStream_t s = (cudaStream_t)stream;
  struct { int st[4]; float loss[3]; } h{};
  static_assert(sizeof(h) == 28, "state block layout");
  YB_CUDA_CHECK(cudaMemcpyAsync(&h, t->val.state, sizeof(h), cudaMemcpyDeviceToHost, s));
  YB_CUDA_CHECK(cudaStreamSynchronize(s));
  if (h.st[1]) { set_error("yb_trainer_val_end: the detection rows overflowed the accumulators"); return YB_ERR_STATE; }
  const int n = h.st[0], m = t->val_labels, nc = t->net.nc, T = VAL_T;
  // ap_per_class outputs: unique | ap | p_curve | r_curve | f1_curve | prec_values | p | r | f1 | tp | fp
  float* o = nullptr;
  const size_t fl = (size_t)nc * (1 + T + 4 * 1000 + 5);
  YB_CUDA_CHECK(cudaMallocAsync((void**)&o, fl * 4, s));
  int* uniq = reinterpret_cast<int*>(o);
  float* ap = o + nc;
  float* curves = ap + (size_t)nc * T;
  float* p = curves + (size_t)nc * 4000;
  float* r = p + nc;
  int counts[3] = {0, 0, 0};
  int rc = yb_ap_per_class(t->val.tp, t->val.conf, t->val.cls, n, T, t->val.target_cls, m, nc, uniq, counts, ap, curves, curves + nc * 1000,
                           curves + nc * 2000, curves + nc * 3000, p, r, r + nc, r + 2 * nc, r + 3 * nc, s);
  std::vector<float> hp(nc), hr(nc), hap((size_t)nc * T);
  const int nu = counts[0];  // classes with labels: rows [0, nu) of the outputs
  if (!rc && (cudaMemcpyAsync(hp.data(), p, (size_t)nu * 4, cudaMemcpyDeviceToHost, s) != cudaSuccess ||
              cudaMemcpyAsync(hr.data(), r, (size_t)nu * 4, cudaMemcpyDeviceToHost, s) != cudaSuccess ||
              cudaMemcpyAsync(hap.data(), ap, (size_t)nu * T * 4, cudaMemcpyDeviceToHost, s) != cudaSuccess ||
              cudaStreamSynchronize(s) != cudaSuccess)) {
    set_error(std::string("yb_trainer_val_end: ") + cudaGetErrorString(cudaGetLastError()));
    rc = YB_ERR_CUDA;
  }
  cudaFreeAsync(o, s);
  if (rc) return rc;
  // P = p.mean(), R = r.mean(), mAP50 = ap[:, 0].mean(), mAP50-95 = ap[:, 1:].mean() (Detector.cs:138-141: the reference's
  // Slice(1) leaves the 0.50 column out of mAP50-95); each mean summed in double and rounded to fp32 once
  double sp = 0, sr = 0, s50 = 0, s95 = 0;
  for (int c = 0; c < nu; c++) {
    sp += hp[c];
    sr += hr[c];
    s50 += hap[(size_t)c * T];
    for (int j = 1; j < T; j++) s95 += hap[(size_t)c * T + j];
  }
  metrics_host[0] = (float)(sp / nu);
  metrics_host[1] = (float)(sr / nu);
  metrics_host[2] = (float)(s50 / nu);
  metrics_host[3] = (float)(s95 / ((double)nu * (T - 1)));
  for (int i = 0; i < 3; i++) loss_items_host[i] = h.loss[i];
  counts_host[0] = t->val_images;
  counts_host[1] = m;
  counts_host[2] = n;
  return YB_OK;
}

int32_t yb_get_grad(yb_trainer* t, const char* name, float* out_host, int64_t count) {
  if (!t || !name || !out_host || !t->net.G) { set_error("yb_get_grad: bad argument"); return YB_ERR_INVALID_ARG; }
  auto it = t->net.pidx.find(name);
  if (it == t->net.pidx.end()) { set_error(std::string("yb_get_grad: unknown parameter ") + name); return YB_ERR_MISSING_WEIGHT; }
  const Entry& e = t->net.params[it->second];
  if (count != e.count) { set_error("yb_get_grad: element count mismatch"); return YB_ERR_SHAPE; }
  YB_CUDA_CHECK(cudaMemcpy(out_host, t->net.G + e.off, (size_t)e.count * sizeof(float), cudaMemcpyDeviceToHost));
  return YB_OK;
}

int32_t yb_get_tensor(yb_trainer* t, const char* name, float* out_host, int64_t count) {
  if (!t || !name || !out_host || !t->net.P) { set_error("yb_get_tensor: bad argument"); return YB_ERR_INVALID_ARG; }
  const Entry* e = nullptr;
  const float* base = nullptr;
  auto it = t->net.pidx.find(name);
  if (it != t->net.pidx.end()) { e = &t->net.params[it->second]; base = t->net.P; }
  else {
    auto is = t->net.sidx.find(name);
    if (is != t->net.sidx.end()) { e = &t->net.stats[is->second]; base = t->net.R; }
  }
  if (!e) { set_error(std::string("yb_get_tensor: unknown tensor ") + name); return YB_ERR_MISSING_WEIGHT; }
  if (count != e->count) { set_error("yb_get_tensor: element count mismatch"); return YB_ERR_SHAPE; }
  YB_CUDA_CHECK(cudaMemcpy(out_host, base + e->off, (size_t)e->count * sizeof(float), cudaMemcpyDeviceToHost));
  return YB_OK;
}

}  // extern "C"
