"""Time the native trainer's eval-mode forward (NativeTrainer.evaluate / yb_trainer_evaluate) on the GPU.

For each model: images/s of `evaluate` at B x 640^2, and `evaluate` against the training step's `yb_train_backward` (train-mode
forward + loss + backward) on the same batch, the two alternated in one process, CUDA events around each call.  Then, in a
profiled pass of its own, the kernels of one call of each: evaluate's kernel time (and the fold launch's share of it)
against the kernel time of the training call's forward part - its kernels before the first loss kernel.  The card's
name, power limit and SM clock limit are read in the same run and printed with the numbers.  Synthetic weights
(tests/util.oracle_model): the time does not depend on the values.

    python tools/exp_eval_time.py [--models v8n,v11s] [--batch 32] [--reps 10]
A model whose activation arena does not fit the card at --batch runs at half that batch (printed)."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else "unknown"


def time_ms(fn, reps):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return sorted(a.elapsed_time(b) for a, b in ev)


def run(model, B, reps):
    from tests.test_train_step import _targets
    from tests.util import oracle_model
    from yolosharp_b200.train_native import NativeTrainer
    from yolosharp_b200 import _lib as L
    import ctypes as C
    arch, size = model[:-1], model[-1]
    sd = oracle_model(arch, "detect", size).state_dict()
    tr = None
    while tr is None:
        try:
            tr = NativeTrainer(sd, arch, size, 80, device="cuda", max_batch=B, height=640, width=640)
        except L.YbError:
            if B == 1:
                raise
            B //= 2
    g = torch.Generator().manual_seed(0)
    x = torch.randint(0, 256, (B, 3, 640, 640), dtype=torch.uint8, generator=g).cuda()
    tg = _targets(B).contiguous()
    sp = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    ev = lambda: tr.evaluate(x)
    bw = lambda: L.check(L.lib().yb_train_backward(tr._h, C.c_void_p(x.data_ptr()), L.YB_U8, B, C.c_void_p(tg.data_ptr()),
                                                    tg.shape[0], None, sp))
    for _ in range(3):  # warm-up of every shape both paths launch
        ev(), bw()
    torch.cuda.synchronize()
    te, tb = [], []
    for _ in range(reps):  # alternated
        te += time_ms(ev, 1)
        tb += time_ms(bw, 1)
    te, tb = sorted(te), sorted(tb)
    med = lambda v: v[len(v) // 2]
    # kernel view, in a pass of its own after the timed window (tracing slows the host): the forward part of the training
    # call is its kernels up to the loss (loss_decode_kernel is the first kernel of v8DetectionLoss)
    ke, kb = kernels(ev), kernels(bw)
    first_loss = next(i for i, k in enumerate(kb) if "loss_decode_kernel" in k[0])
    fwd = kb[:first_loss]
    fold = sum(k[2] - k[1] for k in ke if "tf_fold_all_kernel" in k[0])
    ek, fk = sum(k[2] - k[1] for k in ke), sum(k[2] - k[1] for k in fwd)
    tr.close()
    return {"model": model, "batch": B, "evaluate_ms_median": round(med(te), 3), "evaluate_ms_min": round(te[0], 3),
            "evaluate_images_per_s": round(B / med(te) * 1e3, 1), "train_backward_ms_median": round(med(tb), 3),
            "train_backward_ms_min": round(tb[0], 3), "evaluate_over_train_backward": round(med(te) / med(tb), 3),
            "profiled": {"evaluate_kernel_ms": round(ek / 1e3, 3), "evaluate_span_ms": round((ke[-1][2] - ke[0][1]) / 1e3, 3),
                         "evaluate_kernels": len(ke), "fold_kernel_ms": round(fold / 1e3, 4),
                         "train_forward_kernel_ms": round(fk / 1e3, 3), "train_forward_span_ms": round((fwd[-1][2] - fwd[0][1]) / 1e3, 3),
                         "train_forward_kernels": len(fwd), "evaluate_over_train_forward_kernel_time": round(ek / fk, 3)}}


def kernels(fn):
    """[(name, start_us, end_us)] of the device kernels one call of fn launches, in start order (torch.profiler, CUDA activity)"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ks = [(e.name, e.time_range.start, e.time_range.end)
          for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith(("Memcpy", "Memset"))]
    return sorted(ks, key=lambda k: k[1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="v8n,v11s")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("exp_eval_time.py needs a GPU")
    out = {"card": card(), "results": [run(m, a.batch, a.reps) for m in a.models.split(",")]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
