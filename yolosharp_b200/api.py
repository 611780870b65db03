"""Host-side mirror of the reference's interface for the hot path (same names, argument meaning
and error behaviour), implemented on the C ABI of libyolob200.so:

  reference (C#, /root/reference/YoloSharp)                   here
  ---------------------------------------------------------   -------------------------------
  Models/Yolo.cs:10   Yolo.Yolov8 / Yolov11 / Yolov8Segment   Yolov8 / Yolov11 / Yolov8Segment
  Utils/Ops.cs:239    Ops.non_max_suppression                 Ops.non_max_suppression
  Utils/Ops.cs:462    Ops.process_mask                        Ops.process_mask
  Models/Detector.cs:27 Detector.ImagePredict                 Detector.ImagePredict
  Models/YoloTask.cs:10 YoloTask(Config).LoadModel/ImagePredict  YoloTask
  Types/YoloResult.cs  YoloResult                              YoloResult
  Data/Config.cs       Config (fields used by the path)        Config

There is no CPU implementation here: constructing any of these without an H100 raises.
"""
from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np
import torch

from . import _lib as L
from . import binfmt
from .engine import Engine, masks as _masks, nms as _nms


@dataclass
class YoloResult:
    """Types/YoloResult.cs:3-17."""
    ClassID: int = 0
    Score: float = 0.0
    CenterX: int = 0
    CenterY: int = 0
    Width: int = 0
    Height: int = 0
    Mask: Optional[np.ndarray] = None

    @property
    def X(self):
        return self.CenterX - int(self.Width / 2)

    @property
    def Y(self):
        return self.CenterY - int(self.Height / 2)


@dataclass
class Config:
    """Subset of Data/Config.cs:10-355 read by the predict path (reference defaults)."""
    YoloType: str = "Yolov8"         # Yolov8 | Yolov11
    YoloSize: str = "n"              # n s m l x
    TaskType: str = "Detection"      # Detection | Segmentation
    NumberClass: int = 80
    ImageSize: int = 640
    PredictThreshold: float = 0.3
    IouThreshold: float = 0.7
    ScalarType: str = "Float16"      # Float16 -> tensor-core throughput mode, Float32 -> parity mode
    DeviceIndex: int = 0
    End2End: bool = False            # reference default is true (Config.cs:239); the NMS path needs false
    MaxBatch: int = 1


class _YoloModule:
    """Common part of the graph classes: weights by reference state_dict names, eval-mode forward."""
    arch, task = "v8", "detect"

    def __init__(self, nc=80, reg_max=16, yoloSize="n", end2end=False, device=0, dtype=torch.float16, max_batch=1,
                 flags=0):
        if end2end:
            raise NotImplementedError("end2end heads are not wired into this façade: run the forward and call engine.topk_postprocess "
                                      "(yb_topk_postprocess, Head.cs:117-127) on the decoded prediction tensor")
        if reg_max != 16:
            raise ValueError("reg_max must be 16")
        self.nc, self.yoloSize, self.dtype, self.max_batch, self.flags = nc, yoloSize, dtype, max_batch, flags
        self.device_index = device if isinstance(device, int) else (torch.device(device).index or 0)
        self._state = None
        self._engines = {}
        self.training = False
        L.lib()  # fail here, loudly, if the CUDA library is missing

    # -- torch.nn.Module-like surface used by the reference call sites --
    def eval(self):
        self.training = False
        return self

    def train(self, mode=True):
        if mode:
            raise NotImplementedError("this façade is the inference engine; the training step is yolosharp_b200.train_native.NativeTrainer "
                                      "(yb_train_step) or train.TrainStepV8 / train_v11.TrainStepV11")
        return self

    def load_state_dict(self, state_dict, strict=False):
        """Keys are the reference's (`model.0.conv.weight`, ...).  Returns (missing, unexpected)."""
        self._state = dict(state_dict)
        for e in self._engines.values():
            e.close()
        self._engines = {}
        probe = Engine(self.arch, self.yoloSize, self.task, self.nc, "f32", 0, 1, 64, 64, flags=L.YB_FLAG_DRY_RUN)
        want = probe.expected_tensors()
        probe.close()
        missing = [k for k in want if k not in self._state]
        ws = set(want)
        unexpected = [k for k in self._state if k not in ws]
        if strict and (missing or unexpected):
            raise KeyError(f"missing {missing[:5]}... unexpected {unexpected[:5]}...")
        return missing, unexpected

    def _engine(self, H, W, B, finalize=True):
        key = (H, W)
        e = self._engines.get(key)
        if e is None or e.max_batch < B:
            if e is not None:
                e.close()
            e = Engine(self.arch, self.yoloSize, self.task, self.nc,
                       "f16" if self.dtype == torch.float16 else "f32", self.device_index, max(B, self.max_batch), H, W,
                       self.flags)
            if finalize:
                if self._state is None:
                    raise RuntimeError("no weights loaded: call load_state_dict / LoadModel first "
                                       "(the reference would run with random weights; this engine refuses)")
                e.load_state_dict(self._state)
                e.finalize()
            self._engines[key] = e
        return e

    def forward(self, x, padded_hw=None):
        """Models/Yolo.cs:92-134 in eval mode: returns (inference, preds) with
        inference["boxes"] (B, 4+nc[+32], A) float32 [+ inference["proto"] (B,32,H/4,W/4)].
        padded_hw: run on the input padded right / bottom with 114 to this size (Detector.cs:35-41) without
        materialising the padded tensor."""
        if self.training:
            raise NotImplementedError("train-mode forward")
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"expected (B,3,H,W) input, got {tuple(x.shape)}")
        if not x.is_cuda:
            x = x.to(torch.device("cuda", self.device_index))
        if x.dtype not in (torch.uint8, torch.float16, torch.float32):
            x = x.float()
        x = x.contiguous()
        B, _, H, W = x.shape
        if padded_hw is not None:
            H, W = padded_hw
        e = self._engine(H, W, B)
        if self.task == "segment":
            pred, proto = e.forward(x)
            return {"boxes": pred, "proto": proto}, None
        return {"boxes": e.forward(x)}, None

    __call__ = forward


class Yolov8(_YoloModule):
    arch, task = "v8", "detect"


class Yolov11(_YoloModule):
    arch, task = "v11", "detect"


class Yolov8Segment(_YoloModule):
    arch, task = "v8", "segment"


class Ops:
    @staticmethod
    def non_max_suppression(prediction, conf_thres=0.25, iou_thres=0.45, agnostic=False, max_det=300, nc=0,
                            max_time_img=0.05, max_nms=30000, max_wh=7680, in_place=True, rotated=False,
                            end2end=False):
        """Utils/Ops.cs:239-371.  Returns (output, keepi): per image a (n, 6+extra) tensor
        [x1,y1,x2,y2,conf,cls,extra..] and the kept anchor indices.  `agnostic`, `max_time_img` and
        `in_place` are accepted for signature compatibility (the reference ignores agnostic too; the
        prediction tensor is never modified here)."""
        if conf_thres < 0 or conf_thres > 1:
            raise ValueError(f"Invalid Confidence threshold {conf_thres}, valid values are between 0.0 and 1.0")
        if iou_thres < 0 or iou_thres > 1:
            raise ValueError(f"Invalid IoU {iou_thres}, valid values are between 0.0 and 1.0")
        if rotated or end2end or prediction.shape[-1] == 6:
            raise NotImplementedError("rotated / end2end NMS are outside the accelerated path")
        pred = prediction.float().contiguous()
        dets, counts, keep = _nms(pred, conf_thres, iou_thres, max_det, nc, max_nms, max_wh)
        cnt = counts.tolist()
        output = [dets[i, :cnt[i]] for i in range(len(cnt))]
        keepi = [keep[i, :cnt[i]].long() for i in range(len(cnt))]
        return output, keepi

    @staticmethod
    def process_mask_batch(proto, dets, counts, shape):
        """Batched Utils/Ops.cs:462-489 with upsample=true: -> uint8 (B, max_det, H, W)."""
        return _masks(proto.contiguous(), dets.contiguous(), counts.contiguous(), int(shape[0]), int(shape[1]))


def _to_results(rows):
    """Models/Detector.cs:50-69: truncating conversions; C# integer division truncates toward zero."""
    out = []
    for r in rows.tolist():
        x, y = int(r[0]), int(r[1])
        rw, rh = int(r[2]) - x, int(r[3]) - y
        out.append(YoloResult(ClassID=int(r[5]), Score=float(np.float32(r[4])), CenterX=x + int(rw / 2),
                              CenterY=y + int(rh / 2), Width=rw, Height=rh))
    return out


class Detector:
    """Models/Detector.cs:10-72 (predict side)."""

    def __init__(self, config: Config):
        self.config = config
        dtype = torch.float16 if config.ScalarType == "Float16" else torch.float32
        cls = {"Yolov8": Yolov8, "Yolov11": Yolov11}.get(config.YoloType)
        if cls is None:
            raise NotImplementedError(config.YoloType)
        # note: the reference's Detector ignores Config.YoloSize and always builds size n
        # (Detector.cs:17-20); here the configured size is honoured.
        self.yolo = cls(config.NumberClass, yoloSize=config.YoloSize, end2end=config.End2End,
                        device=config.DeviceIndex, dtype=dtype, max_batch=config.MaxBatch)

    def LoadModel(self, path, skipNcNotEqualLayers=False):
        """Models/YoloBaseTaskModel.cs:27-114.  Unlike the reference a tensor-count mismatch is an
        error, not a silent fall-back to random weights."""
        if skipNcNotEqualLayers:
            raise NotImplementedError("skipNcNotEqualLayers")
        from .engine import read_checkpoint
        sd = {k: v for k, v in read_checkpoint(path).items() if v.dtype.is_floating_point}  # native .bin / .safetensors reader
        missing, _ = self.yolo.load_state_dict(sd)
        if missing:
            raise KeyError(f"{path}: {len(missing)} tensors missing, e.g. {missing[:3]}")

    def ImagePredict(self, orgImage, predictThreshold=None, iouThreshold=None) -> List[YoloResult]:
        """Detector.cs:27-72: uint8 (3,H,W) RGB -> pad right/bottom to x32 with 114 -> /255 -> forward
        -> NMS -> YoloResult list."""
        conf = self.config.PredictThreshold if predictThreshold is None else predictThreshold
        iou = self.config.IouThreshold if iouThreshold is None else iouThreshold
        img = orgImage.to(torch.device("cuda", self.config.DeviceIndex))
        if img.dtype != torch.uint8:
            raise ValueError("ImagePredict expects a uint8 (3,H,W) image tensor")
        x = img.unsqueeze(0).contiguous()
        h, w = x.shape[2], x.shape[3]
        ph, pw = (32 - h % 32) % 32, (32 - w % 32) % 32
        # u8 input: the pad-114 to a multiple of 32 and the /255 are both fused into the first kernel's loads
        inference, _ = self.yolo.eval().forward(x, padded_hw=(h + ph, w + pw))
        out, _ = Ops.non_max_suppression(inference["boxes"], conf, iou)
        return _to_results(out[0].cpu())


class Segmenter(Detector):
    """Models/Segmenter.cs:12-84 (predict side): Detector + Segment head, Proto and instance masks."""

    def __init__(self, config: Config):
        self.config = config
        dtype = torch.float16 if config.ScalarType == "Float16" else torch.float32
        if config.YoloType != "Yolov8":
            raise NotImplementedError("segmentation is built for Yolov8 graphs")
        self.yolo = Yolov8Segment(config.NumberClass, yoloSize=config.YoloSize, end2end=config.End2End,
                                  device=config.DeviceIndex, dtype=dtype, max_batch=config.MaxBatch)

    def ImagePredict(self, orgImage, predictThreshold=None, iouThreshold=None) -> List[YoloResult]:
        """Segmenter.cs:28-84: as Detector.ImagePredict plus process_mask(upsample: true); boxes are
        clipped to the original image (Ops.clip_boxes, Ops.cs:150-158); masks cover the padded input and
        are resized (not cropped) to the original size when padding occurred - the reference's behaviour."""
        conf = self.config.PredictThreshold if predictThreshold is None else predictThreshold
        iou = self.config.IouThreshold if iouThreshold is None else iouThreshold
        img = orgImage.to(torch.device("cuda", self.config.DeviceIndex))
        if img.dtype != torch.uint8:
            raise ValueError("ImagePredict expects a uint8 (3,H,W) image tensor")
        x = img.unsqueeze(0).contiguous()
        h, w = x.shape[2], x.shape[3]
        ph, pw = (32 - h % 32) % 32, (32 - w % 32) % 32
        inference, _ = self.yolo.eval().forward(x, padded_hw=(h + ph, w + pw))
        pred, proto = inference["boxes"], inference["proto"]
        Hp, Wp = h + ph, w + pw  # masks cover the padded input (Segmenter.cs:54)
        dets, counts, _ = _nms(pred, conf, iou, 300, self.config.NumberClass)
        n = int(counts[0].item())
        if n == 0:
            return []
        masks = _masks(proto, dets, counts, Hp, Wp)[0, :n]
        rows = dets[0, :n].clone()
        rows[:, [0, 2]] = rows[:, [0, 2]].clamp(0, w)   # clip_boxes: x to [0, width], y to [0, height]
        rows[:, [1, 3]] = rows[:, [1, 3]].clamp(0, h)
        if ph or pw:
            masks = torch.nn.functional.interpolate(masks[None].float(), size=(h, w), mode="bilinear",
                                                    align_corners=False)[0].to(torch.uint8)
        res = _to_results(rows.cpu())
        mcpu = masks.cpu().numpy()
        for r, mk in zip(res, mcpu):
            r.Mask = mk.T.copy()  # reference stores byte[width, height] (Segmenter.cs:61-62)
        return res


class YoloTask:
    """Models/YoloTask.cs:10-107 (LoadModel / ImagePredict; Train is not built yet)."""

    def __init__(self, config: Config):
        if config.TaskType == "Detection":
            self.yolo = Detector(config)
        elif config.TaskType == "Segmentation":
            self.yolo = Segmenter(config)
        else:
            raise NotImplementedError("Task type not support now.")
        self.config = config

    def LoadModel(self, path, skipNcNotEqualLayers=False):
        self.yolo.LoadModel(path, skipNcNotEqualLayers)

    def Train(self):
        raise NotImplementedError("Train() needs the reference's dataset pipeline (out of scope, DESIGN.md §8); the step it would run per "
                                  "batch is train_native.NativeTrainer.step and the epoch loop is train.fit")

    def ImagePredict(self, image, predictThreshold=None, iouThreshold=None) -> List[YoloResult]:
        if isinstance(image, str):
            import torchvision
            image = torchvision.io.read_image(image, torchvision.io.ImageReadMode.RGB)
        return self.yolo.ImagePredict(image, predictThreshold, iouThreshold)
