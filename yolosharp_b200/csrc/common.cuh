// Shared declarations for the yolob200 engine (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <string>
#include <vector>

#include "yolob200.h"

namespace yb {

// A channel-slice view of an NHWC activation buffer: element (n,h,w,c) lives at
// base[((n*H + h)*W + w) * pitch + coff + c].  Concat/chunk of the reference graph
// (Modules/Block.cs:391-396) become views of one wider buffer - no copies.
struct View {
  void* base = nullptr;  // device pointer to the buffer start (element type = engine storage type)
  int H = 0, W = 0;
  int pitch = 0;  // channels of the whole buffer
  int coff = 0;   // first channel of this view
  int C = 0;      // channels of this view
};

enum Act { ACT_NONE = 0, ACT_SILU = 1 };

// Head-tail fusion (tensor-core path): the final 1x1 convs of the Detect branches write straight into the
// prediction tensor (B, Ctot, A) instead of an NHWC buffer (Modules/Head.cs:204-223 decode).
enum EpiMode { EPI_STORE = 0, EPI_DFL_BOX = 1, EPI_SIGMOID = 2, EPI_RAW = 3 };
struct EpiDecode {
  int mode = EPI_STORE;
  int A = 0, Ctot = 0;  // anchors per image, channels of pred
  int a0 = 0;           // first anchor of this pyramid level
  int ch0 = 0;          // first pred channel written (4 for class probs, 4+nc for mask coeffs)
  int Wl = 0, HW = 0;   // level width, pixels per image
  float stride = 0.f;
};

struct ConvParams {
  View in, out, res;  // res.base == nullptr -> no residual
  View out2;          // optional second destination: nearest-2x upsampled copy (out2.base != nullptr)
  EpiDecode dec;
  int share_sms = 0;  // 1: op runs concurrently with sibling branches - size its grid to half the SMs
  const void* w;      // packed weights, layout depends on kernel
  const float* bias;  // [Cout] fp32 (folded BN beta - mean*scale, or conv bias)
  int B;
  int Cin, Cout;
  int k, stride, pad;
  int Ho, Wo;
  int act;
};

void set_error(const std::string& msg);

#define YB_CUDA_CHECK(expr)                                                                  \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess) {                                                                 \
      ::yb::set_error(std::string(#expr) + " failed: " + cudaGetErrorString(_e) + " at " +   \
                      __FILE__ + ":" + std::to_string(__LINE__));                            \
      return YB_ERR_CUDA;                                                                    \
    }                                                                                        \
  } while (0)

// ---- programmatic dependent launch (PDL) ----
// A kernel launched through launch_pdl may be scheduled while its predecessor in the stream is still running: its CTAs
// become resident as the predecessor's retire, run their prologue (parameter loads, barrier setup, descriptor
// prefetch) and block in pdl_wait() until the predecessor has completed and its writes are visible.  Every kernel of the
// training step calls pdl_wait() before its first global-memory access and pdl_trigger() right AFTER it: the successor
// can be scheduled once all CTAs of this kernel have passed their wait, so at most two kernels of the chain are ever in
// flight (this one finishing, the next one in its prologue).  (Triggering before the wait lets a whole chain of small
// kernels become resident at once; with that form a seven-kernel loss chain read a scalar before its producer's atomics
// - not understood, so the training step uses the conservative order.)  A dependent step of ~800 small kernels otherwise
// pays a drain + launch + fill at every boundary.
// The forward's tensor-core convolutions, fused Bottlenecks and the fp16 SPPF pool (conv_tc.cu, kernels_generic.cu) are
// launched the same way but trigger before their wait, so that the next layer's prologue (weight prefetch) overlaps
// this one's tiles.  YB_NO_PDL=1 launches all of these kernels the ordinary way (A/B measurements).
// Both instructions are no-ops in a kernel launched the ordinary way, so a kernel may be launched either way.
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
bool pdl_enabled();  // false when YB_NO_PDL is set (A/B measurements)
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(static_cast<Args&&>(args))...);
}

// storage type <-> fp32 for the kernels templated on T = float | __half
template <typename T> __device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<__half>(__half v) { return __half2float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __half from_f<__half>(float v) { return __float2half_rn(v); }

// SiLU, x * sigmoid(x) written as x / (1 + exp(-x)) like ATen's silu kernel: ONE definition for the fp32 CUDA-core
// kernels, the BatchNorm apply passes of bn_train.cu and the eval epilogue of tf_conv_kernel, so that they round alike
__device__ __forceinline__ float silu_f(float u) { return u / (1.f + expf(-u)); }
#endif

// ---- kernels_generic.cu : CUDA-core kernels, templated on storage type (float | __half) ----
template <typename T>
int launch_conv_generic(const ConvParams& p, cudaStream_t s);
template <typename T>
int launch_dwconv3x3(const ConvParams& p, cudaStream_t s);  // depthwise 3x3 s1 p1, w [9][C] fp32
template <typename T>
int launch_sppf_pool(const View& in, const View& out5, const View& out9, const View& out13, int B,
                     cudaStream_t s);
template <typename T>
int launch_upsample2x(const View& in, const View& out, int B, cudaStream_t s);
// network input (B,3,H,W) NCHW of dtype u8/f16/f32 -> NHWC T with pitch/coff from `out`
template <typename T>
int launch_input_to_nhwc(const void* in, int in_dtype, const View& out, int B, cudaStream_t s, int src_H = 0, int src_W = 0);
// read back a view as NCHW fp32 (debug)
template <typename T>
int launch_view_to_nchw_f32(const View& in, float* out, int B, cudaStream_t s);

// Head decode (Modules/Head.cs:204-223 + Block.cs:15-45 + Tal.cs:313-356):
// box logits (64 ch) + class logits (nc ch) [+ mask coeffs] of one level, NHWC ->
// rows [0,4) xywh*stride, [4,4+nc) sigmoid, [4+nc,..) coeffs of pred (B, Ctot, A), anchors
// [a0, a0 + H*W) of this level.
template <typename T>
int launch_decode_level(const View& box, const View& cls, const View* coef, int B, int nc, int nm,
                        int reg_max, float stride, int a0, int A, int Ctot, float* pred,
                        cudaStream_t s);
template <typename T>
int launch_pixel_shuffle2(const View& in, const View& out, int B, cudaStream_t s);
// proto (B,h,w,32) NHWC T -> (B,32,h,w) fp32
template <typename T>
int launch_proto_out(const View& in, float* out, int B, cudaStream_t s);

// ---- conv_tc.cu : wgmma implicit-GEMM conv (fp16 storage, fp32 accumulate) ----
// Device queries, cached after the first call: the driver's cuTensorMapEncodeTiled (nullptr when the entry point is
// missing) and the SM count of the current device (one value per device).
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn tmap_encode_fn();
int sm_count();
// 4-D tensor map {C, W, H, N} of an NHWC buffer of `type` (FLOAT16 or FLOAT32) elements whose pixels are `pitch` channels
// apart, starting at channel coff
CUresult tmap_nhwc(CUtensorMap* map, CUtensorMapDataType type, void* base, int coff, int C, int W, int H, int N, int pitch,
                   const cuuint32_t* box, const cuuint32_t* estr, CUtensorMapSwizzle swz);
// Dynamic shared-memory limit of `kernel` on the current device for a launch of `smem` bytes, and for the persistent
// ring kernels (max_carveout) the largest carveout.  Every kernel whose launch needs more than 48 KiB sets its limit
// here.  Launches of different sizes share a kernel: its limit (per device) only ever grows to the largest launch so far,
// so a smaller launch set up later cannot make an earlier one fail.  cudaFuncSetAttribute acts on the current device only,
// so the limit is kept per (device, kernel).
cudaError_t smem_limit(const void* kernel, size_t smem, bool max_carveout);
struct TcConvPlan;  // opaque: tensor maps + tiling for one conv layer
TcConvPlan* tc_conv_plan_create(const ConvParams& p, std::string* err);
void tc_conv_plan_destroy(TcConvPlan* plan);
std::string tc_conv_plan_describe(const TcConvPlan* plan);  // tiling summary (YB_DEBUG_PLANS)
int tc_conv_launch(const TcConvPlan* plan, int B, float* pred, int* tile_ctr, cudaStream_t s);
bool tc_conv_supported(const ConvParams& p);
// Fused Bottleneck (DESIGN 4.1): the 3x3 conv `pa` and the 3x3 conv `pb` that reads its output (plus the shortcut
// `pb` may carry) as one launch; the intermediate stays in shared memory.  Uses both plans' packed weights, so they must
// outlive it.  nullptr (and *err) when the pair's shapes do not fit the kernel.
struct TcBneckPlan;
TcBneckPlan* tc_bneck_plan_create(const TcConvPlan* pa, const TcConvPlan* pb, std::string* err);
void tc_bneck_plan_destroy(TcBneckPlan* plan);
std::string tc_bneck_plan_describe(const TcBneckPlan* plan);
int tc_bneck_launch(const TcBneckPlan* plan, int B, int* tile_ctr, cudaStream_t s);
// Folded 1x1 (DESIGN 4.1): the conv `pa` and the 1x1 conv `pb` that is the only reader of its output as one
// conv_tc_kernel launch; `pa`'s activations go from its accumulator to `pb`'s MMA in registers and are never stored.
// The result is an ordinary plan (tc_conv_launch / describe / destroy) that uses both plans' packed weights, so they
// must outlive it.  nullptr (and the reason in *err) when the pair does not fit.
TcConvPlan* tc_fold_plan_create(const TcConvPlan* pa, const TcConvPlan* pb, std::string* err);
// stem: NCHW u8/f16/f32 input -> 3x3 s2 conv (Cin=3) + bias + SiLU -> NHWC fp16
int launch_stem_f16(const void* in, int in_dtype, int B, int H, int W, const __half* w16 /*[Cout][32]*/,
                    const float* bias, const View& out, cudaStream_t s, int src_H = 0, int src_W = 0);  // src_*: unpadded source size

// ---- nms.cu ----
int nms_launch(const float* pred, int B, int C, int A, int nc, float conf, float iou, int max_det,
               int max_nms, int max_wh, float* dets, int* counts, int* keep_idx, cudaStream_t s);
int detection_loss_launch(const float* boxes, const float* scores, int B, int nc, int reg_max, int H, int W,
                          const float* targets_host, int n_targets, int topk, float hyp_box, float hyp_cls, float hyp_dfl,
                          float* loss_items, float* grad_boxes, float* grad_scores, unsigned char* fg_out, int* gt_idx_out,
                          float* tscore_out, cudaStream_t s);
// counters: optional >= 64 zeroed words owned by ONE stream (the statistics kernels leave them zero); nullptr = allocate and
// clear per call
int bn_silu_train_forward(const float* z, long long M, int C, int pitch, const float* gamma, const float* beta, float eps,
                          float momentum, int act, float* running_mean, float* running_var, float* y, int ypitch,
                          float* save_mean, float* save_invstd, cudaStream_t s, unsigned* counters = nullptr);
// the elementwise pass alone: y = act(gamma * (z - mean) * invstd + beta) (eval mode: mean / invstd from the running statistics)
int bn_silu_apply(const float* z, long long M, int C, int pitch, const float* mean, const float* invstd, const float* gamma,
                  const float* beta, int act, float* y, int ypitch, cudaStream_t s);
int bn_silu_backward(const float* z, const float* dy, long long M, int C, int pitch, int dpitch, const float* gamma,
                     const float* beta, const float* save_mean, const float* save_invstd, int act, float* dz, int zpitch,
                     float* dgamma, float* dbeta, cudaStream_t s, unsigned* counters = nullptr);
int adamw_step(float* p, const float* g, float* m, float* v, long long n, int step, float lr, float b1, float b2, float eps,
               float wd, cudaStream_t s);
int conv_backward_data(const float* dz, const float* w, int N, int H, int W, int Cin, int Cout, int k, int stride, int pad,
                       float* dx, cudaStream_t s);
int conv_backward_weight(const float* x, const float* dz, int N, int H, int W, int Cin, int Cout, int k, int stride, int pad,
                         float* dw, cudaStream_t s);
int masks_launch(const float* proto, const float* dets, const int* counts, int B, int max_det, int nm,
                 int mh, int mw, int H, int W, uint8_t* masks, cudaStream_t s, int mask_cap = 0);  // mask_cap: masks per image (0 = max_det)
// false (and the error set) when no CUDA device is present: the C entry points' first check.  ndev: the device count.
bool have_device(const char* who, int* ndev = nullptr);

// ---- attention.cu : C2PSA attention core (limits: key_dim <= 64, head_dim <= 128, N <= 6 012 tokens at 32 / 64) ----
// engine: qkv (B,N,nh*(2kd+hd)) -> out (B,N,nh*hd) and the dense v copy for the pe conv
template <typename T>
int launch_attention(const View& qkv, const View& out, const View& vout, int B, int nh, int kd, int hd, float scale,
                     cudaStream_t s);
// training, fp32: q, k (B, N, nh, kd); v, out, dout (B, N, nh, hd); row_max / row_sum optional (B, nh, N)
int attention_forward_f32(const float* q, const float* k, const float* v, int B, int N, int nh, int kd, int hd, float scale,
                          float* out, float* row_max, float* row_sum, cudaStream_t s);
int attention_backward_f32(const float* q, const float* k, const float* v, const float* dout, int B, int N, int nh, int kd,
                           int hd, float scale, float* dq, float* dk, float* dv, cudaStream_t s);

// ---- entry points of the native training step (train_step.cu) in the other translation units ----
// conv_tf32.cu : TF32 tensor-core convolutions
int tf_conv_forward(const float* x, const float* w, const float* bias, int N, int H, int W, int Cin, int Cout, int k, int stride,
                    int pad, float* z, float* ws, size_t ws_bytes, cudaStream_t s, int x_pitch, const float* prepacked,
                    std::string* desc = nullptr);
int tf_conv_backward_data(const float* dz, const float* w, int N, int H, int W, int Cin, int Cout, int k, int stride, int pad,
                          float* dx, float* ws, size_t ws_bytes, cudaStream_t s, const float* prepacked,
                          std::string* desc = nullptr);
int tf_conv_backward_weight(const float* x, const float* dz, int N, int H, int W, int Cin, int Cout, int k, int stride, int pad,
                            float* dw, float* ws, size_t ws_bytes, cudaStream_t s, int x_pitch, std::string* desc = nullptr);
size_t tf_conv_workspace_bytes(int N, int H, int W, int Cin, int Cout, int k, int stride);
struct TfPackDesc { long long off, chunk0; int cout, cin, taps, pad_; };  // off: element offset in the flat buffers; chunk0: first block
long long tf_pack_chunks(int cout, int cin, int taps);
int tf_pack_all(const float* P, float* WF, float* WB, const TfPackDesc* dev_descs, int nd, long long total_chunks, cudaStream_t s);
// eval mode: BatchNorm (running statistics, eps 1e-3) folded into one conv's forward B operand and bias.  gamma == nullptr:
// a plain Conv2d, weights packed unscaled; wf == nullptr: per-channel vectors only (bias, invstd: each optional)
struct TfFoldDesc {
  const float *w, *gamma, *beta, *rm, *rv;
  float *wf, *bias, *invstd;
  long long chunk0;  // first block of this descriptor
  int cout, cin, taps, pad_;
};
long long tf_fold_chunks(const TfFoldDesc& d);
int tf_fold_all(const TfFoldDesc* dev_descs, int nd, long long total_chunks, cudaStream_t s);
// eval-mode Conv block on wf (the folded [tap][Cout][Cin] operand): out[.., out_coff + c] = [res +] act(conv(x) + bias), on
// channel-slice views (pitches in elements, multiples of 4, 16-byte aligned bases)
int tf_conv_forward_eval(const float* x, int x_pitch, const float* wf, const float* bias, int N, int H, int W, int Cin, int Cout, int k,
                         int stride, int act, const float* res, int res_pitch, float* out, int out_pitch, int out_coff, cudaStream_t s,
                         std::string* desc = nullptr);
int stem3_forward(const float* x, int xc, const float* w, int N, int H, int W, int C, float* z, cudaStream_t s);
int stem3_backward_weight(const float* x, int xc, const float* dz, int N, int H, int W, int C, float* dw, float* ws, size_t ws_bytes,
                          cudaStream_t s);
// loss.cu
int detection_loss_prepare(const float* targets_host, int n_targets, int B, int nc, int H, int W, std::vector<float>& gts, int* n_max_out);
int detection_loss_launch_dev(const float* boxes, const float* scores, int B, int nc, int reg_max, int H, int W, const float* d_gts,
                              int n_max, int topk, float hyp_box, float hyp_cls, float hyp_dfl, float* loss_items, float* grad_boxes,
                              float* grad_scores, unsigned char* fg_out, int* gt_idx_out, float* tscore_out, cudaStream_t s);
// val.cu : the per-batch tail of the trainer's validation pass (NMS -> labels -> matching -> append) and its accumulators
// Detector.Val's max_det and IoU thresholds linspace(0.5, 0.95, 10); labels per batch: the matching kernel's shared arrays
constexpr int VAL_MAX_DET = 300, VAL_T = 10, VAL_MAX_BATCH_LABELS = 2048;
struct ValAccum {
  unsigned char* tp;  // (cap_rows, VAL_T) correct bits
  float* conf;        // (cap_rows)
  int* cls;           // (cap_rows) predicted class
  int* target_cls;    // (max_labels)
  int* state;         // [0] rows appended so far, [1] overflow flag
  float* loss;        // [3] summed loss items
  long long cap_rows;
};
int val_batch_launch(const float* pred, int B, int nc, int A, int H, int W, const float* rows, int n_labels, long long label_off,
                     const float* loss_detach, float* labels, float* dets, int* counts, unsigned char* correct, const ValAccum& acc,
                     cudaStream_t s);
int val_append_launch(const unsigned char* tp, const float* conf, const int* pred_cls, int n, const int* target_cls, int m,
                      long long label_off, const ValAccum& acc, cudaStream_t s);
// train_v11.cu : depthwise 3x3, stride 1, pad 1, fp32 NHWC
int dwconv3x3_forward_f32(const float* x, const float* w, int N, int H, int W, int C, float* z, cudaStream_t s);
int dwconv3x3_backward_f32(const float* x, const float* dz, const float* w, int N, int H, int W, int C, float* dx, float* dw,
                           cudaStream_t s);

}  // namespace yb
