/*
 * yolob200.h - C ABI of the H100-native YOLO forward / NMS engine.
 *
 * This is the drop-in boundary for the hot path of IntptrMax/YoloSharp (reference
 * @16dc3cd, paths below relative to /root/reference/YoloSharp).  The reference has no
 * FFI of its own; these entry points are what a C# `[DllImport("yolob200")]` shim (see
 * INTEGRATION.md) binds in place of the TorchSharp calls at the seams listed per function.
 *
 * Conventions
 *   - plain C types only; every function returns 0 (YB_OK) or a negative yb_status and never
 *     throws; the message for the last failure on the calling thread is yb_last_error().
 *   - "dev" pointers are CUDA device pointers on the engine's device; the caller (TorchSharp /
 *     PyTorch tensors) owns all input/output buffers, the engine owns weights + workspace.
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).
 *   - one engine = one device, not re-entrant (the reference runs the model on the caller's
 *     thread only, Models/YoloBaseTaskModel.cs:19).
 */
#ifndef YOLOB200_H
#define YOLOB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define YB_ABI_VERSION 1

typedef enum {
  YB_OK = 0,
  YB_ERR_INVALID_ARG = -1,   /* reference: ArgumentException (e.g. Utils/Ops.cs:248-255) */
  YB_ERR_NOT_IMPLEMENTED = -2, /* reference: NotImplementedException */
  YB_ERR_CUDA = -3,
  YB_ERR_STATE = -4,         /* call order violated (e.g. forward before finalize) */
  YB_ERR_MISSING_WEIGHT = -5,
  YB_ERR_SHAPE = -6,
  YB_ERR_NO_DEVICE = -7
} yb_status;

/* Types/YoloTypes.cs: YoloType / YoloSize / TaskType */
typedef enum { YB_ARCH_V8 = 8, YB_ARCH_V11 = 11 } yb_arch;
typedef enum { YB_SIZE_N = 0, YB_SIZE_S = 1, YB_SIZE_M = 2, YB_SIZE_L = 3, YB_SIZE_X = 4 } yb_size;
typedef enum { YB_TASK_DETECT = 0, YB_TASK_SEGMENT = 1 } yb_task;

/* arithmetic mode of the network body */
typedef enum {
  YB_PREC_F32 = 0, /* parity mode: fp32 storage + fp32 FMA (matches the fp32 oracle to ~1e-5) */
  YB_PREC_F16 = 1  /* throughput mode: fp16 NHWC storage, wgmma tensor-core MMA, fp32 accumulate */
} yb_precision;

/* element types of caller buffers; values are torch ScalarType codes as stored in the
 * reference's .bin checkpoints (Utils/Lib.cs:38) */
typedef enum { YB_U8 = 0, YB_F16 = 5, YB_F32 = 6, YB_BF16 = 15 } yb_dtype;

typedef struct {
  int32_t arch;       /* yb_arch   - Data/Config.cs YoloType */
  int32_t size;       /* yb_size   - Data/Config.cs YoloSize (Models/Yolo.cs:45-49, 213-217) */
  int32_t task;       /* yb_task */
  int32_t nc;         /* number of classes (Config.NumberClass, default 80) */
  int32_t reg_max;    /* DFL bins, 16 */
  int32_t precision;  /* yb_precision */
  int32_t device;     /* CUDA device ordinal */
  int32_t max_batch;  /* workspace is planned for this many images */
  int32_t height;     /* input H, multiple of 32 (Models/Detector.cs:35-41 pads to it) */
  int32_t width;      /* input W, multiple of 32 */
  int32_t flags;      /* YB_FLAG_* */
} yb_config;

#define YB_FLAG_NO_TCGEN05 1  /* F16 mode: use the CUDA-core fp16 kernels instead of the tensor-core kernels (debug) */
#define YB_FLAG_NO_GRAPH   2  /* do not capture the forward into a CUDA graph */
#define YB_FLAG_NO_CONCURRENCY 8  /* run the independent head branches serially on one stream */
#define YB_FLAG_DRY_RUN    4  /* build the op graph / expected-tensor list only (no CUDA calls; for host-side checks).
                                 Every compute entry point fails with YB_ERR_STATE on such an engine. */

typedef struct yb_engine yb_engine;

/* ABI / build info. */
int32_t yb_abi_version(void);
const char* yb_build_info(void);
const char* yb_last_error(void);

/* Replaces: `new Yolo.Yolov8(nc, yoloSize:..)` / `Yolov11` / `Yolov8Segment` construction
 * (Models/Yolo.cs:27-39, 204-207, 339-342; Models/Detector.cs:12-25). */
int32_t yb_create(const yb_config* cfg, yb_engine** out);
void yb_destroy(yb_engine* e);

/* Number of anchors A and channels of the prediction tensor for the configured input size:
 * pred is (B, 4+nc[+32], A) as produced by Detect._inference (Modules/Head.cs:204-208). */
int32_t yb_num_anchors(const yb_engine* e);
int32_t yb_pred_channels(const yb_engine* e);

/* Replaces: `yolo.load_state_dict(state_dict)` (Models/YoloBaseTaskModel.cs:100).  `name` is a
 * reference state_dict key (e.g. "model.0.conv.weight", "model.22.cv2.0.2.bias"); `data` is a
 * HOST pointer to `ndim`-shaped row-major data of `dtype` (YB_F16 / YB_F32 / YB_BF16).
 * Unknown names (num_batches_tracked, anchors, strides, dfl.conv.weight) are accepted and ignored. */
int32_t yb_load_tensor(yb_engine* e, const char* name, int32_t dtype, int32_t ndim,
                       const int64_t* shape, const void* data);

/* Native checkpoint ingest (csrc/ckpt.cu; host code, no TorchSharp / PyTorch needed).
 * Replaces: `Lib.LoadModel` for the TorchSharp `.bin` format (Utils/Lib.cs:9-54), `SafetensorsLoader`
 * (ModelLoader/SafetensorsLoader.cs:7-109), `PickleLoader` for torch.save archives (ModelLoader/PickleLoader.cs:21-466: zip +
 * pickle; tensors are named by their path through dicts / lists / object attributes, a pickled nn.Module yields its
 * state_dict() names - an Ultralytics checkpoint gives "model.model.0.conv.weight", ...) and `SaveWeight`
 * (Models/YoloBaseTaskModel.cs:470-490).  The format is chosen by the file extension (`.safetensors`, `.pt` / `.pth`,
 * anything else = `.bin`).  dtype codes are torch ScalarType values (yb_dtype; also 1 i8, 2 i16, 3 i32, 4 i64, 7 f64, 11 bool).
 *   yb_load_checkpoint  = open + yb_load_tensor for every f16 / f32 / bf16 tensor; when no name of the file is an expected
 *                         name but the names are after dropping a leading "model." (an Ultralytics {'model': object}
 *                         checkpoint), that level is dropped (+ counts of loaded tensors and of
 *                         expected tensors the file lacks; unlike YoloBaseTaskModel.cs:32-35 nothing falls back to
 *                         random weights: yb_finalize_weights fails on the first missing tensor)
 *   yb_ckpt_*           iterate a file without an engine; pointers stay valid until yb_ckpt_close */
typedef struct yb_ckpt yb_ckpt;
int32_t yb_ckpt_open(const char* path, yb_ckpt** out);
int32_t yb_ckpt_count(const yb_ckpt* c);
int32_t yb_ckpt_tensor(const yb_ckpt* c, int32_t i, const char** name, int32_t* dtype, int32_t* ndim, const int64_t** shape,
                       const void** data, int64_t* nbytes);
void yb_ckpt_close(yb_ckpt* c);
int32_t yb_load_checkpoint(yb_engine* e, const char* path, int32_t* n_loaded, int32_t* n_missing);
int32_t yb_ckpt_write_bin(const char* path, int32_t count, const char* const* names, const int32_t* dtypes, const int32_t* ndims,
                          const int64_t* const* shapes, const void* const* datas);

/* Fold eval-mode BatchNorm (eps 1e-3, Modules/Convs.cs:41) into the conv weights, pack to the
 * device layouts, build TMA descriptors.  Fails with YB_ERR_MISSING_WEIGHT naming the first
 * absent tensor (the reference silently keeps random weights, YoloBaseTaskModel.cs:32-35; we do not). */
int32_t yb_finalize_weights(yb_engine* e);

/* Number of parameter/buffer tensors the engine expects, and their names (for host-side checks). */
int32_t yb_num_expected_tensors(const yb_engine* e);
const char* yb_expected_tensor_name(const yb_engine* e, int32_t i);

/* Replaces: `yolo.forward(input).inference["boxes"]` [+ `["proto"]`] in eval mode
 * (Models/Yolo.cs:92-134 -> Modules/Head.cs:89-115, 283-306).
 *   in       dev, NCHW (B,3,H,W): YB_F32/YB_F16 already scaled to [0,1] (Detector.cs:41),
 *            or YB_U8 raw pixels (the /255 is fused into the stem)
 *   out_pred dev, float32 (B, 4+nc[+32], A): xywh in input pixels, class probabilities, mask coeffs
 *   out_proto dev, float32 (B,32,H/4,W/4) for segment engines, else NULL */
int32_t yb_forward(yb_engine* e, const void* in, int32_t in_dtype, int32_t batch,
                   float* out_pred, float* out_proto, void* stream);

/* yb_forward on images that are NOT yet padded to the planned size: `in` is (B,3,src_height,src_width) contiguous with
 * src <= the engine's height / width, and the right / bottom padding with the value 114 that `Detector.ImagePredict`
 * applies before the /255 (Models/Detector.cs:35-41: pad to a multiple of 32) is produced inside the first kernel
 * (the stem's loads) instead of by a separate pad pass.  Float inputs must already be scaled to [0,1] (the padded
 * pixels are 114/255). */
int32_t yb_forward_padded(yb_engine* e, const void* in, int32_t in_dtype, int32_t batch, int32_t src_height, int32_t src_width,
                          float* out_pred, float* out_proto, void* stream);

/* Replaces: `Ops.non_max_suppression(prediction, conf_thres, iou_thres, .., max_det, nc, ..,
 * max_nms, max_wh)` (Utils/Ops.cs:239-371), non-rotated, non-end2end path, incl. the
 * torchvision.ops.nms call at :357.
 *   pred     dev, float32 (B, C, A) with C = 4 + nc + extra (not modified: the reference's
 *            in-place xywh->xyxy conversion is done on the fly)
 *   dets     dev, float32 (B, max_det, 6+extra): x1,y1,x2,y2,conf,cls,extra.. score-descending;
 *            rows >= counts[b] are zero
 *   counts   dev, int32 (B)
 *   keep_idx dev, int32 (B, max_det) original anchor index of each kept row (`keepi`), or NULL
 * Errors: conf/iou outside [0,1] -> YB_ERR_INVALID_ARG (reference throws ArgumentException). */
int32_t yb_nms(const float* pred, int32_t batch, int32_t channels, int32_t anchors, int32_t nc,
               float conf_thres, float iou_thres, int32_t max_det, int32_t max_nms, int32_t max_wh,
               float* dets, int32_t* counts, int32_t* keep_idx, void* stream);

/* Replaces (training path, first step): `v8DetectionLoss.forward` (Utils/Loss.cs:328-485) incl. the
 * TaskAlignedAssigner (Utils/Tal.cs:13-311, topk = 10, alpha 0.5, beta 6), BboxLoss/DFLoss (Loss.cs:94-167) and the
 * CIoU of Utils/Metrics.cs:36-111, on the raw outputs of the train-mode head (Head.cs:71-87):
 *   boxes   dev float32 (B, 4*reg_max, A) distribution logits;  scores dev float32 (B, nc, A) class logits
 *   height/width  network input size (anchor grid = strides 8/16/32, Tal.cs:313-335)
 *   targets HOST float32 (n_targets, 6) rows [image index, class, x, y, w, h] with xywh normalised to [0,1]
 *           (= cat(batch_idx, cls, bboxes), Loss.cs:424)
 *   loss_items  dev float32 (3): box, cls, dfl after the gains = the reference's `loss.detach()` (Loss.cs:473)
 *   grad_boxes / grad_scores  dev, same shapes as boxes / scores, or NULL: gradient of sum(loss_items) * B, i.e. of
 *           the tensor the reference calls backward on (Loss.cs:473 returns loss * batch_size)
 *   fg / gt_idx / target_score  optional dev outputs (B, A): uint8 foreground flag, int32 assigned target row inside
 *           the image, float32 normalised alignment score - for tests and for the mask / pose losses later
 * The assignment is computed from detached values, as in the reference. */
int32_t yb_detection_loss(const float* boxes, const float* scores, int32_t batch, int32_t nc, int32_t reg_max,
                          int32_t height, int32_t width, const float* targets_host, int32_t n_targets, int32_t topk,
                          float hyp_box, float hyp_cls, float hyp_dfl, float* loss_items, float* grad_boxes,
                          float* grad_scores, uint8_t* fg, int32_t* gt_idx, float* target_score, void* stream);

/* Replaces (training path): BatchNorm2d in TRAIN mode followed by SiLU inside every `Conv` block
 * (Modules/Convs.cs:36-56 under `yolo.train()`, YoloBaseTaskModel.cs:299,325; BatchNorm2d(eps 1e-3, momentum 0.03)).
 *   z       dev float32, M = B*H*W rows x C channels, row pitch `pitch` elements (NHWC conv output)
 *   y       dev float32 (M, C) with row pitch `ypitch`: act ? SiLU(bn(z)) : bn(z)
 *   running_mean / running_var  dev (C), updated in place with `momentum` and the UNBIASED batch variance, or NULL
 *   save_mean / save_invstd     dev (C) outputs the backward pass needs */
int32_t yb_bn_silu_train_forward(const float* z, int64_t rows, int32_t channels, int32_t pitch, const float* gamma,
                                 const float* beta, float eps, float momentum, int32_t act, float* running_mean,
                                 float* running_var, float* y, int32_t ypitch, float* save_mean, float* save_invstd,
                                 void* stream);
/* Backward of the above: dy (M, C) -> dz (M, C), dgamma (C), dbeta (C). */
int32_t yb_bn_silu_backward(const float* z, const float* dy, int64_t rows, int32_t channels, int32_t pitch,
                            int32_t dpitch, const float* gamma, const float* beta, const float* save_mean,
                            const float* save_invstd, int32_t act, float* dz, int32_t zpitch, float* dgamma,
                            float* dbeta, void* stream);
/* Replaces: one `AdamW.step()` over a flat parameter group (YoloBaseTaskModel.cs:142-160 builds
 * AdamW(lr = round(0.01/(4+nc), 6), weight_decay 5e-4, default betas 0.9 / 0.999, eps 1e-8); Utils/Amp.cs:260-286
 * calls it).  p, g, m, v: dev float32 (n); step counts from 1. */
int32_t yb_adamw_step(float* p, const float* g, float* m, float* v, int64_t n, int32_t step, float lr, float beta1,
                      float beta2, float eps, float weight_decay, void* stream);

/* Replaces (training path, fp32 parity kernels): the forward of `Conv2d` without the (train-mode) BatchNorm folded in
 * (Modules/Convs.cs:44, Head.cs:41-52 for the biased 1x1 convs).
 *   x  dev float32 NHWC (N, H, W, Cin);  w_packed dev float32 [kh][kw][Cin][Cout] (= weight.permute(2,3,1,0));
 *   bias dev float32 (Cout) or NULL;  z dev float32 NHWC (N, Ho, Wo, Cout) */
int32_t yb_conv_forward_f32(const float* x, const float* w_packed, const float* bias, int32_t n, int32_t height,
                            int32_t width, int32_t cin, int32_t cout, int32_t k, int32_t stride, int32_t pad, float* z,
                            void* stream);
/* Replaces (training path, fp32 parity kernels): the autograd backward of `Conv2d(bias: false)` inside every Conv
 * block (Modules/Convs.cs:44; libtorch dgrad / wgrad behind `loss.backward()`, Utils/Amp.cs:260-286).
 *   x  dev float32 NHWC (N, H, W, Cin);  dz dev float32 NHWC (N, Ho, Wo, Cout), Ho = (H + 2 pad - k)/stride + 1
 *   w  dev float32 in the checkpoint layout (Cout, Cin, k, k);  dx like x;  dw like w */
int32_t yb_conv_backward_data(const float* dz, const float* w, int32_t n, int32_t height, int32_t width, int32_t cin,
                              int32_t cout, int32_t k, int32_t stride, int32_t pad, float* dx, void* stream);
int32_t yb_conv_backward_weight(const float* x, const float* dz, int32_t n, int32_t height, int32_t width, int32_t cin,
                                int32_t cout, int32_t k, int32_t stride, int32_t pad, float* dw, void* stream);

/* Replaces (training path, tensor cores): the same three convolution passes as the fp32 parity kernels above -
 * `Conv2d.forward` and the dgrad / wgrad libtorch runs behind `loss.backward()` (Modules/Convs.cs:44,
 * Utils/Amp.cs:260-286) - as tensor-core implicit GEMMs with TF32 operands and fp32 accumulation (the arithmetic class of
 * libtorch's own CUDA convolutions, whose cuDNN path allows TF32 by default).  Same tensors and layouts as
 * yb_conv_forward_f32 / yb_conv_backward_*, except that `w` is always the checkpoint layout (Cout, Cin, k, k).
 * Supported: cin % 8 == 0, cout % 8 == 0, k in {1, 3}, stride in {1, 2}, pad == k / 2 (stride-2 dgrad: even height /
 * width); anything else returns YB_ERR_SHAPE and the caller uses the fp32 kernels (the 3-channel stem).
 *   workspace  dev scratch of at least yb_conv_tc_workspace_bytes(...) bytes (re-packed weights / split-K partials of
 *              the weight gradient); may be shared by all calls of one stream. */
int64_t yb_conv_tc_workspace_bytes(int32_t n, int32_t height, int32_t width, int32_t cin, int32_t cout, int32_t k,
                                   int32_t stride);
int32_t yb_conv_forward_tc(const float* x, const float* w, const float* bias, int32_t n, int32_t height, int32_t width,
                           int32_t cin, int32_t cout, int32_t k, int32_t stride, int32_t pad, float* z, void* workspace,
                           int64_t workspace_bytes, void* stream);
int32_t yb_conv_backward_data_tc(const float* dz, const float* w, int32_t n, int32_t height, int32_t width, int32_t cin,
                                 int32_t cout, int32_t k, int32_t stride, int32_t pad, float* dx, void* workspace,
                                 int64_t workspace_bytes, void* stream);
int32_t yb_conv_backward_weight_tc(const float* x, const float* dz, int32_t n, int32_t height, int32_t width, int32_t cin,
                                   int32_t cout, int32_t k, int32_t stride, int32_t pad, float* dw, void* workspace,
                                   int64_t workspace_bytes, void* stream);

/* The 3-channel stem of the training step (model.0 = Conv(3, C, k 3, s 2), Models/Yolo.cs:53) in fp32 on CUDA cores: one
 * K = 3 x 9 contraction per output is too thin for a tensor-core tile (the padded-to-8 TF32 form was bound by the TMA row
 * rate).  x dev float32 NHWC with `x_channels` >= 3 channels per pixel (the first 3 are read); w (C, 3, 3, 3) checkpoint
 * layout; z / dz (N, H/2, W/2, C); C % 8 == 0, C <= 128, even H and W; workspace >= yb_conv_tc_workspace_bytes(...). */
int32_t yb_stem_conv_forward_f32(const float* x, int32_t x_channels, const float* w, int32_t n, int32_t height, int32_t width,
                                 int32_t cout, float* z, void* stream);
int32_t yb_stem_conv_backward_weight_f32(const float* x, int32_t x_channels, const float* dz, int32_t n, int32_t height,
                                         int32_t width, int32_t cout, float* dw, void* workspace, int64_t workspace_bytes,
                                         void* stream);

/* Replaces: `AMPWrapper.TrainStep` (Utils/Amp.cs:260-286: yolo.forward -> loss -> loss.backward() -> optimizer.step()) for
 * the YOLOv8 / YOLOv11 detect models as ONE call (csrc/train_step.cu): train-mode forward with batch-statistics
 * BatchNorm, v8DetectionLoss, backward through the whole graph (TF32 tensor-core convolutions), AdamW per name group
 * (YoloBaseTaskModel.cs:142-160: the "bias" group first).
 *   yb_trainer_create   cfg: arch (8 | 11), size, nc, device, max_batch, height, width (task detect);
 *                       flags & YB_FLAG_DRY_RUN builds the parameter layout only (no device memory)
 *   yb_trainer_tensor_info  kind 0: trained parameters, kind 1: BatchNorm running statistics; names are the reference's
 *                       state_dict keys, offset / count locate the tensor in the flat buffer of its kind
 *   yb_trainer_flat_size    kind 0: floats of the parameter buffers, 1: of the running-statistics buffer,
 *                       2: floats of the leading "bias" group inside the parameter buffers
 *   yb_trainer_bind     the caller owns the flat fp32 device buffers (parameters, gradients, Adam m / v, running stats):
 *                       a TorchSharp / PyTorch host wraps them as tensors, loads a checkpoint into them, reads gradients
 *                       and all-reduces the gradient buffer between yb_train_backward and yb_train_apply (DDP)
 *   yb_train_backward   images dev (B, 3, H, W) u8 (scaled by 1/255 as the training loader does, Data/YoloDataset.cs:140) or
 *                       f32; targets HOST float32 (n, 6) rows [image, class, x, y, w, h] normalised, staged to the device
 *                       before the forward pass is queued (the call does not synchronise until the end); loss_items HOST
 *                       float[3] (the call then returns after the stream has finished) or NULL (fully asynchronous).
 *                       A trainer is driven from ONE stream at a time (its activation arena, packed-weight buffers and
 *                       BatchNorm ticket counters belong to the step in flight).
 *   yb_train_apply      one AdamW step (betas 0.9 / 0.999, eps 1e-8) with the two group learning rates
 *   yb_train_step       = yb_train_backward + yb_train_apply (single device)
 *   yb_get_grad / yb_get_tensor  copy one named gradient / parameter / running statistic to the host
 *   yb_trainer_evaluate `AMPWrapper.Evaluate` (Utils/Amp.cs:387-395: the training model in `eval()`, its prediction
 *                       `inference["boxes"]` and the raw head outputs `preds`): an eval-mode forward of the trainer's own
 *                       graph at its current parameters and running statistics, in the training arithmetic (TF32
 *                       tensor-core convolutions, fp32 storage).  BatchNorm uses the running statistics, folded into each
 *                       dense conv's weights and bias (one fold launch per call); every Conv block is one conv launch.
 *                       images as yb_train_backward, 1 <= batch <= max_batch at the trainer's height x width.  Device
 *                       outputs, each optional (NULL: not written): pred (B, 4 + nc, A) decoded boxes xywh + class
 *                       probabilities, boxes (B, 64, A) and scores (B, nc, A) the raw head outputs v8DetectionLoss reads.
 *                       Asynchronous on `stream`; touches no parameter, running statistic, gradient, Adam moment or
 *                       BatchNorm ticket counter (it shares the activation arena with the step: one stream at a time). */
typedef struct yb_trainer yb_trainer;
int32_t yb_trainer_create(const yb_config* cfg, yb_trainer** out);
void yb_trainer_destroy(yb_trainer* t);
int32_t yb_trainer_num_tensors(const yb_trainer* t, int32_t kind);
int32_t yb_trainer_tensor_info(const yb_trainer* t, int32_t kind, int32_t index, const char** name, int64_t* offset,
                               int64_t* count, int32_t* ndim, const int64_t** shape);
int64_t yb_trainer_flat_size(const yb_trainer* t, int32_t kind);
int32_t yb_trainer_bind(yb_trainer* t, float* params, float* grads, float* adam_m, float* adam_v, float* running_stats);
int32_t yb_train_backward(yb_trainer* t, const void* images, int32_t in_dtype, int32_t batch, const float* targets_host,
                          int32_t n_targets, float* loss_items_host, void* stream);
int32_t yb_train_apply(yb_trainer* t, float lr_bias, float lr_other, float weight_decay, void* stream);
int32_t yb_train_step(yb_trainer* t, const void* images, int32_t in_dtype, int32_t batch, const float* targets_host,
                      int32_t n_targets, float lr_bias, float lr_other, float weight_decay, float* loss_items_host,
                      void* stream);
int32_t yb_get_grad(yb_trainer* t, const char* name, float* out_host, int64_t count);
int32_t yb_get_tensor(yb_trainer* t, const char* name, float* out_host, int64_t count);
int32_t yb_trainer_evaluate(yb_trainer* t, const void* images, int32_t in_dtype, int32_t batch, float* pred, float* boxes,
                            float* scores, void* stream);
/* The trainer's validation pass, `Detector.Val` (Models/Detector.cs:73-160) over a loader, on the device.
 *   yb_trainer_val_begin   sizes trainer-owned accumulators (outside the activation arena) for at most max_images x 300
 *                          detection rows and max_labels labels, and resets the rows, loss sums and image / label counts
 *   yb_trainer_val_batch   one loader iteration (Detector.cs:81-132), images and targets as yb_train_backward: the eval
 *                          forward of yb_trainer_evaluate, v8DetectionLoss without gradients added to the loss sums,
 *                          non_max_suppression(conf 0.1, iou 0.7, max_det 300, max_nms 30000, max_wh 7680), the labels
 *                          `xywh2xyxy(bboxes * (w, h, w, h))`, match_predictions at linspace(0.5, 0.95, 10) and the append of
 *                          every image's kept rows (tp bits, conf, class) in image order.  Queued on `stream` without a host
 *                          wait other than for the pinned target buffer (as yb_train_backward).  n_targets == 0: the batch is
 *                          skipped (Detector.cs:91-94).  YB_ERR_INVALID_ARG for batch > max_batch, a class id outside
 *                          [0, nc), more than 2048 labels in the batch, or more images / labels than val_begin was sized for;
 *                          YB_ERR_STATE before val_begin.
 *   yb_trainer_val_append  appends device rows in the accumulator layout: tp uint8 (n, 10), conf float32 (n), pred_cls
 *                          int32 (n), target_cls int32 (m); the loss sums and the image count are not touched.  With
 *                          yb_trainer_val_rows this merges the rows of data-parallel ranks before val_end.
 *   yb_trainer_val_rows    HOST counts_host[2] = accumulated rows n and labels m (synchronises `stream`); when the device
 *                          pointers are given (capacity n / m) the rows are copied there in the layout val_append takes;
 *                          clear != 0 then empties the rows and labels (the loss sums and the image count stay)
 *   yb_trainer_val_end     ap_per_class on the accumulated rows; synchronises.  HOST outputs: loss_items[3] the SUM of the
 *                          executed batches' loss items (the reference's fitness is -sum of them); metrics[4] = P, R, mAP50,
 *                          mAP50-95 with P = p.mean(), R = r.mean() over the classes that have labels, mAP50 = ap[:, 0].mean()
 *                          and mAP50-95 = ap[:, 1:].mean() - the reference's Slice(1) leaves the 0.50 column out (Detector.cs:141);
 *                          each mean summed in double and rounded to float32 once.  counts[3] = images, labels, detection rows.
 *                          YB_ERR_STATE when no labels were accumulated (the reference's torch.cat of empty lists throws)
 *                          or the rows overflowed.  Calling it again returns the same numbers.
 * The pass changes no parameter, running statistic, gradient, Adam moment or BatchNorm ticket counter; like the step it is
 * driven from one stream at a time. */
int32_t yb_trainer_val_begin(yb_trainer* t, int32_t max_images, int32_t max_labels, void* stream);
int32_t yb_trainer_val_batch(yb_trainer* t, const void* images, int32_t in_dtype, int32_t batch, const float* targets_host,
                             int32_t n_targets, void* stream);
int32_t yb_trainer_val_append(yb_trainer* t, const uint8_t* tp, const float* conf, const int32_t* pred_cls, int32_t n,
                              const int32_t* target_cls, int32_t m, void* stream);
int32_t yb_trainer_val_rows(yb_trainer* t, uint8_t* tp, float* conf, int32_t* pred_cls, int32_t* target_cls, int32_t* counts_host,
                            int32_t clear, void* stream);
int32_t yb_trainer_val_end(yb_trainer* t, float* loss_items_host, float* metrics_host, int32_t* counts_host, void* stream);

/* Replaces (training path of YOLOv11, fp32 parity kernels): the forward and the autograd backward of the depthwise 3x3
 * convolutions - `Convs.DWConv` (Modules/Convs.cs:108-114; groups = gcd(c1, c2) = c for every use in Yolov11: the
 * class branch of the head, Head.cs:50, and `Attention.pe`, Block.cs:746), stride 1, padding 1.
 *   x, z, dz, dx  dev float32 NHWC (N, H, W, C);  w, dw  dev float32 (C, 1, 3, 3) checkpoint layout */
int32_t yb_dwconv3x3_forward_f32(const float* x, const float* w, int32_t n, int32_t height, int32_t width, int32_t channels,
                                 float* z, void* stream);
int32_t yb_dwconv3x3_backward_f32(const float* x, const float* dz, const float* w, int32_t n, int32_t height, int32_t width,
                                  int32_t channels, float* dx, float* dw, void* stream);
/* Replaces (training path of YOLOv11): the attention core of `Block.Attention.forward` (Modules/Block.cs:785-809):
 * out[b, i, h, :] = sum_j softmax_j(scale * q[b, i, h, :] . k[b, j, h, :]) v[b, j, h, :], and its backward.
 *   q, k, dq, dk  dev float32 (B, N, heads, key_dim);  v, out, dout, dv  dev float32 (B, N, heads, head_dim)
 * Limits (forward and backward): key_dim <= 64, head_dim <= 128, and 8 N + 32 (key_dim + 1) + 32 head_dim floats
 * <= 200 KiB, i.e. N <= 6012 tokens at key_dim 32, head_dim 64 (YOLOv11 up to 2464 x 2464); beyond them
 * YB_ERR_SHAPE with the limit in yb_last_error(). */
int32_t yb_attention_forward_f32(const float* q, const float* k, const float* v, int32_t batch, int32_t tokens, int32_t heads,
                                 int32_t key_dim, int32_t head_dim, float scale, float* out, void* stream);
int32_t yb_attention_backward_f32(const float* q, const float* k, const float* v, const float* dout, int32_t batch, int32_t tokens,
                                  int32_t heads, int32_t key_dim, int32_t head_dim, float scale, float* dq, float* dk, float* dv,
                                  void* stream);

/* Replaces: `Ops.process_mask(proto[i], rows[:,6:], rows[:,:4], shape, upsample:true)`
 * (Utils/Ops.cs:462-489, CUDA branch of crop_mask :437-447) for a whole batch.
 *   proto  dev float32 (B,32,mh,mw);  dets/counts as written by yb_nms with extra == 32
 *   masks  dev uint8 (B, max_det, H, W), 1 where mask > 0; rows >= counts[b] untouched */
int32_t yb_masks(const float* proto, const float* dets, const int32_t* counts, int32_t batch,
                 int32_t max_det, int32_t nm, int32_t mh, int32_t mw, int32_t height, int32_t width,
                 uint8_t* masks, void* stream);

/* Replaces: the body of `Detector.ImagePredict` (Models/Detector.cs:27-72) for a batch of
 * equally sized images: HOST uint8 (B,3,H,W) RGB in, HOST detections out; H2D copy, /255,
 * forward, NMS and D2H copy run on `stream` and the call returns after the results landed.
 *   dets_host   float32 (B, max_det, 6[+32]);  counts_host int32 (B) */
int32_t yb_predict_u8(yb_engine* e, const uint8_t* images_host, int32_t batch, float conf_thres,
                      float iou_thres, int32_t max_det, float* dets_host, int32_t* counts_host,
                      void* stream);

/* Pipelined form of yb_predict_u8 for serving loops: `slot` (0 .. 3) selects one of four engine-owned
 * stream + staging-buffer sets, so the H2D copy / forward / NMS / D2H of one batch overlap those of the
 * others (the forwards themselves are serialised on the shared activation arena).  submit returns immediately; the host buffers must stay valid (and should be pinned) until
 * yb_predict_u8_wait(slot) returned. */
int32_t yb_predict_u8_submit(yb_engine* e, int32_t slot, const uint8_t* images_host, int32_t batch,
                             float conf_thres, float iou_thres, int32_t max_det, float* dets_host,
                             int32_t* counts_host);
int32_t yb_predict_u8_wait(yb_engine* e, int32_t slot);

/* Replaces: the body of `Segmenter.ImagePredict` (Models/Segmenter.cs:28-84) for a batch of equally sized images on a
 * segment engine: as yb_predict_u8_submit, plus the instance masks of the first `mask_cap` kept detections of every
 * image (score order) - `Ops.process_mask(.., upsample: true)` - copied to the host.
 *   dets_host   float32 (B, max_det, 38);  counts_host int32 (B)
 *   masks_host  uint8 (B, mask_cap, H, W), 1 where mask > 0; planes >= min(counts[b], mask_cap) are not written
 * Wait with yb_predict_u8_wait(slot). */
int32_t yb_predict_seg_u8_submit(yb_engine* e, int32_t slot, const uint8_t* images_host, int32_t batch, float conf_thres,
                                 float iou_thres, int32_t max_det, int32_t mask_cap, float* dets_host, int32_t* counts_host,
                                 uint8_t* masks_host);

/* Replaces: `Detect.postprocess` + `Detect.get_topk_index` (Modules/Head.cs:117-127, 175-196) - the NMS-free tail an
 * end2end head runs instead of non_max_suppression (`Config.End2End` defaults to true, Data/Config.cs:239): the
 * k = min(max_det, A) anchors with the largest best-class score, then the k largest of their k x nc class scores.
 *   pred  dev float32 (B, channels >= 4 + nc, A), channel-major as written by yb_forward (rows 0-3 xywh, then scores)
 *   out   dev float32 (B, k, 6) rows [x, y, w, h, score, class], score-descending;  idx  dev int32 (B, k) anchor of
 *         every row, or NULL;  agnostic != 0 = the `agnostic_nms` branch (one row per selected anchor, its best class).
 * Equal scores are taken in index order (torch.topk leaves that choice unspecified).  max_det <= 1024. */
int32_t yb_topk_postprocess(const float* pred, int32_t batch, int32_t channels, int32_t anchors, int32_t nc,
                            int32_t max_det, int32_t agnostic, float* out, int32_t* idx, void* stream);

/* Decode tails of the OBB and Pose heads and the rotated NMS (csrc/heads.cu), fp32.
 * yb_obb_decode   replaces `Obb._inference` (Modules/Head.cs:410-436 on top of Detect._inference :204-223): DFL expectation
 *                 of box_logits (B, 4*reg_max, A), angle = (sigmoid(angle_logits (B,1,A)) - 0.25) * pi, `Tal.dist2rbox`
 *                 (Utils/Tal.cs:389-408) with anchors (2, A) / strides (A), class sigmoid -> out (B, 4 + nc + 1, A)
 * yb_pose_decode  replaces `Pose.kpts_decode` (Modules/Head.cs:595-609): kpts (B, nk, A) -> out, keypoint_dim 2 or 3
 * yb_probiou      replaces `Metrics.batch_probiou` (Utils/Metrics.cs:223-254): xywhr (n, 5) x (m, 5) -> (n, m)
 * yb_nms_rotated  replaces `Ops.nms_rotated(boxes, scores, threshold)` (Utils/Ops.cs:373-401, use_triu): keep (n) int32
 *                 receives the kept original indices in score order, count (1) their number. All pointers device. */
int32_t yb_obb_decode(const float* box_logits, const float* cls_logits, const float* angle_logits, const float* anchors,
                      const float* strides, int32_t batch, int32_t anchors_n, int32_t nc, int32_t reg_max, float* out,
                      void* stream);
int32_t yb_pose_decode(const float* kpts, const float* anchors, const float* strides, int32_t batch, int32_t anchors_n,
                       int32_t nk, int32_t keypoint_dim, float* out, void* stream);
int32_t yb_probiou(const float* obb1, int32_t n, const float* obb2, int32_t m, float eps, float* out, void* stream);
int32_t yb_nms_rotated(const float* boxes, const float* scores, int32_t n, float threshold, int32_t* keep, int32_t* count,
                       void* stream);

/* Validation-side post-processing (csrc/val.cu), batched over the images of a step.
 * yb_box_iou  replaces `Metrics.box_iou(box1, box2)` (Utils/Metrics.cs:16-34): out (n, m) float32, xyxy boxes.
 * yb_match_predictions  replaces the per-image `match_predictions(pred_classes, true_classes, iou)` loop of
 * `Detector.Val` (Models/YoloBaseTaskModel.cs:377-446, Models/Detector.cs:103-120):
 *   dets / counts  as written by yb_nms (B, max_det, row_width) / (B)
 *   labels  dev float32 (n_labels, 6) rows [image, class, x1, y1, x2, y2] in input pixels (batch_idx, cls, xywh2xyxy(bboxes * scale))
 *   iou_thresholds_host  the reference's linspace(0.5, 0.95, 10) as float32 (HOST pointer)
 *   correct  dev uint8 (B, max_det, n_thresholds): 1 where detection d is a true positive at threshold i */
int32_t yb_box_iou(const float* box1, int32_t n, const float* box2, int32_t m, float eps, float* out, void* stream);
/* yb_mask_iou  replaces `Metrics.mask_iou(mask1, mask2)` (Utils/Metrics.cs:120-125, called by Segmenter.Val, Models/Segmenter.cs:142):
 * mask1 (n1, pixels), mask2 (n2, pixels) float32 flattened masks -> out (n1, n2) float32. */
int32_t yb_mask_iou(const float* mask1, int32_t n1, const float* mask2, int32_t n2, int32_t pixels, float eps, float* out, void* stream);

int32_t yb_match_predictions(const float* dets, const int32_t* counts, int32_t batch, int32_t max_det, int32_t row_width,
                             const float* labels, int32_t n_labels, const float* iou_thresholds_host, int32_t n_thresholds,
                             uint8_t* correct, void* stream);

/* Replaces `Metrics.ap_per_class(tp, conf, pred_cls, target_cls)` (Utils/Metrics.cs:308-384, with compute_ap :395-421,
 * interp :424-468 and smooth :475-487), the reduction `Detector.Val` runs over ALL detections of a validation pass
 * (csrc/metrics.cu).  Where the reference's three unstable `torch.argsort` calls meet equal keys its result is unspecified;
 * this entry point uses the stable order (ties keep their input order).
 *   tp  dev uint8 (n, n_thresholds) as yb_match_predictions writes it (rows of real detections only), conf dev float32 (n),
 *   pred_cls dev int32 (n), target_cls dev int32 (m), classes in [0, max_classes), max_classes <= 4096
 *   unique_classes dev int32 (max_classes): the classes that have labels, ascending (the reference's torch.unique)
 *   counts_host  HOST int32[3]: number of unique classes nc, rows of prec_values (classes with labels AND predictions),
 *                index of the best smoothed-F1 point
 *   ap dev (max_classes, n_thresholds); p_curve / r_curve / f1_curve / prec_values dev (max_classes, 1000);
 *   p, r, f1, tp_out, fp_out dev (max_classes): rows [0, nc) are written as the reference returns them.
 * The call synchronises the stream (it returns counts).
 * yb_linspace01  torch.linspace(0, 1, steps) as ATen computes it (the `x` axis the reference also returns), HOST output. */
int32_t yb_ap_per_class(const uint8_t* tp, const float* conf, const int32_t* pred_cls, int32_t n, int32_t n_thresholds,
                        const int32_t* target_cls, int32_t m, int32_t max_classes, int32_t* unique_classes, int32_t* counts_host,
                        float* ap, float* p_curve, float* r_curve, float* f1_curve, float* prec_values, float* p, float* r, float* f1,
                        float* tp_out, float* fp_out, void* stream);
int32_t yb_linspace01(int32_t steps, float* out_host);

/* The instance-mask term of `v8SegmentationLoss` (Utils/Loss.cs:688-865: `calculate_segmentation_loss` :806-861 with
 * `single_mask_loss` :787-795, overlap_mask = true), loss and gradients (csrc/segloss.cu).  The box / cls / dfl terms and the
 * assignment are yb_detection_loss's (the criterion derives from v8DetectionLoss, :411-468); this entry point takes
 *   fg (B, A) uint8, gt_idx (B, A) int32       as yb_detection_loss returns them
 *   target_bboxes (B, A, 4)                     the assigned ground-truth boxes, xyxy in input pixels
 *   masks (B, mask_h, mask_w) float32           instance index + 1 per pixel, 0 = background (the reference's overlap encoding)
 *   proto (B, nm, mask_h, mask_w), mask_coefficient (B, nm, A)   the Segment head's train-mode outputs (nm <= 64)
 *   img_h, img_w                                the input size (feats[0] shape * stride[0], :744)
 * and writes loss_item (1) = loss[1] after the `hyp_box` gain (the value the criterion reports), grad_proto and
 * grad_coefficient = d(loss[1] * batch) / d(proto, mask_coefficient) (the criterion returns loss * batch_size, :785).
 * All pointers device.  Masks at another resolution than proto (the reference's interpolate branch, :739-743) are not
 * supported. */
int32_t yb_segmentation_loss(const uint8_t* fg, const int32_t* gt_idx, const float* target_bboxes, const float* masks,
                             const float* proto, const float* mask_coefficient, int32_t batch, int32_t anchors, int32_t nm,
                             int32_t mask_h, int32_t mask_w, float img_h, float img_w, float hyp_box, float* loss_item,
                             float* grad_proto, float* grad_coefficient, void* stream);

/* ---- multi-GPU: exchange of the fixed-capacity detection payloads over NVLink peer memory (csrc/comm.cu) ----
 * Design target SURVEY.md section 8(e); the reference is single-device (Data/Config.cs:301), so this surface is
 * net-new.  One yb_comm per process (= per GPU), all ranks on one node.  Every rank pushes its payload into a
 * window of every peer with plain stores through cudaIpc-mapped pointers and publishes a sequence flag; consumers
 * poll flags in their own memory - no collective kernel has to be co-resident on all ranks.
 *   1. yb_comm_create on every rank (same world / bytes_per_rank / slots)
 *   2. yb_comm_local_handle -> exchange the yb_comm_handle_bytes() opaque bytes by any host channel
 *      (torch.distributed, MPI, files) -> yb_comm_connect with all ranks' handles in rank order
 *   3. per step: producer kernels write the payload into yb_comm_send_buffer(slot); yb_comm_allgather(slot, stream);
 *      after it (stream order) yb_comm_window(slot) holds world x bytes_per_rank, rank r at offset r * bytes_per_rank;
 *      yb_comm_release(slot, stream) once the consumer is done (peers may then overwrite the slot). */
typedef struct yb_comm yb_comm;
int32_t yb_comm_handle_bytes(void);
int32_t yb_comm_create(int32_t rank, int32_t world, int32_t device, int64_t bytes_per_rank, int32_t slots, yb_comm** out);
int32_t yb_comm_local_handle(yb_comm* c, void* handle_out);
int32_t yb_comm_connect(yb_comm* c, const void* handles /* world x yb_comm_handle_bytes(), rank order */);
int32_t yb_comm_info(const yb_comm* c, int32_t* rank, int32_t* world, int64_t* bytes_per_rank, int32_t* slots);
void* yb_comm_send_buffer(yb_comm* c, int32_t slot);
void* yb_comm_window(yb_comm* c, int32_t slot);
int32_t yb_comm_allgather(yb_comm* c, int32_t slot, void* stream);
int32_t yb_comm_release(yb_comm* c, int32_t slot, void* stream);
void yb_comm_destroy(yb_comm* c);
/* bytes of one rank's detection payload: dets (batch, max_det, row_width) float32 followed by counts (batch) int32,
 * each padded to 16 bytes - the layout yb_predict_u8_submit_gather and bench.py use */
int64_t yb_comm_detection_payload_bytes(int32_t batch, int32_t max_det, int32_t row_width);

/* yb_predict_u8_submit for a batch sharded over `world` GPUs (BASELINE configs[2]): as yb_predict_u8_submit, but the
 * NMS rows of every rank are exchanged through `comm` slot `slot` before the D2H copy, so all_dets_host
 * (world*batch, max_det, 6[+32]) / all_counts_host (world*batch) receive the detections of ALL ranks in global
 * image order.  Every rank must call it with the same batch / max_det; wait with yb_predict_u8_wait(slot). */
int32_t yb_predict_u8_submit_gather(yb_engine* e, yb_comm* comm, int32_t slot, const uint8_t* images_host, int32_t batch,
                                    float conf_thres, float iou_thres, int32_t max_det, float* all_dets_host,
                                    int32_t* all_counts_host);

/* Debug / profiling helpers (not part of the reference surface). */
int32_t yb_num_ops(const yb_engine* e);
/* copy the activation written by op `op_index` (NHWC -> NCHW float32 host buffer); returns
 * channels*H*W per image through *chw (C,H,W) */
int32_t yb_debug_read_activation(yb_engine* e, int32_t op_index, int32_t batch, float* host_out,
                                 int64_t host_capacity, int32_t chw[3]);
const char* yb_op_name(const yb_engine* e, int32_t op_index);
/* number of kernel launches one yb_forward issues (for bench.py's gpu_launches) */
int32_t yb_launches_per_forward(const yb_engine* e);
/* Per-op timing: runs the forward eagerly (no graph) with a CUDA event pair around every op on
 * `stream`; ms_per_op[i] (i < yb_num_ops) receives the device time of op i. */
int32_t yb_profile_forward(yb_engine* e, const void* in, int32_t in_dtype, int32_t batch, float* out_pred,
                           float* out_proto, float* ms_per_op, int32_t n_ops, void* stream);
/* Back-to-back timing of ONE op: `reps` launches of op `op_index` between two CUDA events on `stream`, on the data
 * the last forward left in the engine's buffers (launch gaps amortised; used by bench.py to take the non-conv
 * kernels out of the graph-timed forward when it reports the dominant kernel's in-graph time). */
int32_t yb_time_op(yb_engine* e, int32_t op_index, const void* in, int32_t in_dtype, int32_t batch, float* out_pred,
                   float* out_proto, int32_t reps, float* ms_per_launch, void* stream);
/* Algorithmic work of op i for `batch` images: flops = 2*MACs (convs only), bytes = input view +
 * output view (+ residual) + weights, each counted once (SURVEY.md section 8(d) definitions).  An op fused into the
 * next op's launch reports the bytes of that launch there: the first conv of a fused Bottleneck keeps its FLOPs and
 * reports 0 bytes; a conv folded into a 1x1 reports 0 FLOPs and 0 bytes, and the 1x1 reports both convs' FLOPs and
 * the producer's input, both weight sets and its own output. */
int32_t yb_op_cost(const yb_engine* e, int32_t op_index, int32_t batch, double* flops, double* bytes);
/* 0 = tensor-core conv, 1 = CUDA-core conv, 2 = stem, 3 = depthwise, 4 = pool, 5 = upsample, 7 = other;
 * 6 = launches nothing of its own and reports no FLOPs or bytes: a fused Detect decode, or a conv folded into the next
 * op's 1x1 launch (that op reports the FLOPs of both convs and the bytes its launch moves) */
int32_t yb_op_kind(const yb_engine* e, int32_t op_index);
/* debug: the `skip`-th tensor-core conv launch from now records a clock64 timeline of CTA 0 into dev_buf (128 x int64) */
int32_t yb_debug_timeline(long long* dev_buf, int32_t skip);
/* debug: ONE launch of the fp16 tensor-core convolution (conv_tc_kernel) on caller-owned device buffers, planned as the
 * engine plans its layers; synchronises before it returns.  Op-level tests compare it with a float64 convolution.
 *   in      fp16 NHWC (plan_batch, height, width, in_pitch), the input channels at [in_coff, in_coff + cin)
 *   w       fp16 [cout][k][k][cin];  bias float32 (cout);  k 1 (stride 1) or 3 (stride 1 or 2), pad k / 2;  act 0 / 1 (SiLU)
 *   res     fp16 (plan_batch, Ho, Wo, res_pitch) added after the activation at [res_coff, ..), or NULL
 *   out     fp16 (plan_batch, Ho, Wo, out_pitch), written at [out_coff, out_coff + cout); NULL with a decode epilogue
 *   plan_batch / run_batch  images the plan is made for / launched with (run_batch <= plan_batch)
 *   share_sms   1: the grid trimming of a layer that shares the GPU with a sibling head branch
 *   tile_counter  1: dynamic tile queue, 0: static round-robin tile order
 *   dec_*   fused Detect epilogue of a 1x1 conv (dec_mode 1 DFL box, 2 sigmoid, 3 raw; 0 = store into out): pred float32
 *           (run_batch, dec_channels, dec_anchors) receives anchors dec_a0 .. dec_a0 + dec_pixels - 1 of a level dec_width
 *           pixels wide, channels dec_ch0 .. (rows 0-3 for the box), box coordinates times dec_stride
 *   desc    receives the plan description (tc_conv_plan_describe), or NULL
 * A shape the tensor-core conv or its planner does not take returns YB_ERR_SHAPE with the reason. */
int32_t yb_debug_conv_f16(const void* in, int32_t plan_batch, int32_t run_batch, int32_t height, int32_t width, int32_t in_pitch,
                          int32_t in_coff, int32_t cin, const void* w, const float* bias, int32_t cout, int32_t k, int32_t stride,
                          int32_t act, const void* res, int32_t res_pitch, int32_t res_coff, void* out, int32_t out_pitch,
                          int32_t out_coff, int32_t share_sms, int32_t tile_counter, int32_t dec_mode, int32_t dec_anchors,
                          int32_t dec_channels, int32_t dec_a0, int32_t dec_ch0, int32_t dec_width, int32_t dec_pixels,
                          float dec_stride, float* pred, char* desc, int32_t desc_capacity);
/* debug: ONE launch of the fused Bottleneck kernel (bneck_tc_kernel) on caller-owned device buffers: out = SiLU(conv_b(t) +
 * bias_b) [+ x], t = fp16(SiLU(conv_a(x) + bias_a)), both 3x3 stride 1; synchronises before it returns.
 *   x       fp16 NHWC (batch, height, width, x_pitch), channels [x_coff, x_coff + cin); also the shortcut when shortcut != 0
 *   w_a     fp16 [cmid][3][3][cin], bias_a float32 (cmid);  w_b fp16 [cout][3][3][cmid], bias_b float32 (cout)
 *   out     fp16 (batch, height, width, out_pitch), written at [out_coff, out_coff + cout)
 *   desc    receives the fused plan's description (tc_bneck_plan_describe), or NULL
 * A pair the fused kernel does not take returns YB_ERR_SHAPE with the planner's reason. */
int32_t yb_debug_bneck_f16(const void* x, int32_t batch, int32_t height, int32_t width, int32_t x_pitch, int32_t x_coff, int32_t cin,
                           const void* w_a, const float* bias_a, int32_t cmid, const void* w_b, const float* bias_b, int32_t cout,
                           int32_t shortcut, void* out, int32_t out_pitch, int32_t out_coff, char* desc, int32_t desc_capacity);

/* debug: ONE pass of the TF32 tensor-core training convolution (csrc/conv_tf32.cu) on caller-owned device buffers, through
 * the same host functions the training step calls; synchronises before it returns.  Op-level tests compare it with a
 * float64 convolution.  k 1 or 3, stride 1 or 2, pad k / 2, cin and cout multiples of 8.
 *   pass 0  forward:          out (n, Ho, Wo, cout) = conv(x, w) + bias (bias may be NULL)
 *   pass 1  data gradient:    out (n, height, width, cin) = dx from dz (n, Ho, Wo, cout); height, width even at stride 2
 *   pass 2  weight gradient:  out (cout, cin, k, k) = dw from x and dz
 *   x       fp32 NHWC (n, height, width, cin); x_pitch 0 = dense, else the element stride between pixels, x pointing at the
 *           first channel of the view (16-byte aligned, x_pitch a multiple of 4); passes 0 and 2 only
 *   w       fp32 (cout, cin, k, k), the checkpoint layout;  workspace: yb_conv_tc_workspace_bytes(...) bytes
 *   desc    receives one line per kernel launch with the values that were launched (tf_conv_kernel: BK, chunks,
 *           n_tile x n_tiles, BW x BH, in_stride, flat, ntaps, occ, stages, grid; tf_wgrad_kernel: halo, tpc, nb,
 *           co_tiles, ci_tiles, co_blocks, splits, pix_tiles, b_stages, grid), or NULL
 * A shape the kernels or their planners do not take returns YB_ERR_SHAPE with the reason. */
int32_t yb_debug_conv_tf32(int32_t pass, const float* x, int32_t x_pitch, const float* dz, const float* w, const float* bias,
                           int32_t n, int32_t height, int32_t width, int32_t cin, int32_t cout, int32_t k, int32_t stride,
                           float* out, void* workspace, int64_t workspace_bytes, char* desc, int32_t desc_capacity);
/* debug: the eval sibling of yb_debug_conv_tf32 - ONE fold launch and ONE eval-mode conv launch of the Conv block in `eval()`
 * (Modules/Convs.cs:36-56: SiLU(BatchNorm2d(conv(x))) with the running statistics, eps 1e-3), through the host functions
 * yb_trainer_evaluate calls; synchronises before it returns.
 *   out[.., out_coff + c] = [res +] act(conv(x, folded_w) + folded_bias),  act 0 = identity, 1 = SiLU
 *   x          fp32 NHWC (n, height, width, *), x_pitch 0 = dense (cin), else the element stride between pixels
 *   w          fp32 (cout, cin, k, k) checkpoint layout; gamma, beta, running_mean, running_var fp32 (cout)
 *   res        NULL or fp32 NHWC (n, Ho, Wo, *) view added after the activation (the Bottleneck shortcut, Block.cs:606);
 *              res_pitch 0 = dense (cout)
 *   out        fp32 NHWC (n, Ho, Wo, out_pitch), written at channels [out_coff, out_coff + cout) only
 *   folded_w   receives the folded forward operand [k * k][cout][cin]: w * gamma / sqrt(rv + 1e-3), computed in double and
 *              rounded to fp32 once;  folded_bias receives (cout) beta - rm * gamma / sqrt(rv + 1e-3), likewise
 *   desc       receives the conv launch's description line (as yb_debug_conv_tf32, kernel name tf_conv_kernel_eval), or NULL
 * Pitches and out_coff must be multiples of 4 on 16-byte aligned views; k 1 or 3, stride 1 or 2, cin and cout multiples of 8. */
int32_t yb_debug_conv_tf32_eval(const float* x, int32_t x_pitch, const float* w, const float* gamma, const float* beta,
                                const float* running_mean, const float* running_var, int32_t n, int32_t height, int32_t width,
                                int32_t cin, int32_t cout, int32_t k, int32_t stride, int32_t act, const float* res, int32_t res_pitch,
                                float* out, int32_t out_pitch, int32_t out_coff, float* folded_w, float* folded_bias, char* desc,
                                int32_t desc_capacity);

#ifdef __cplusplus
}
#endif
#endif /* YOLOB200_H */
