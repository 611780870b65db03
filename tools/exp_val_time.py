"""Time one call of the trainer's validation pass (yb_trainer_val_batch) against one eval-mode forward (yb_trainer_evaluate)
on the GPU.

For each model at B x 640^2, u8 images, synthetic weights (tests/util.oracle_model: a few hundred NMS survivors per image):
the median of `--reps` calls of each, alternated in one process, CUDA events around each call.  Then, in a profiled pass of
its own, the kernels of one val_batch call: the share of its first-to-last-kernel span taken by everything after the
forward (loss + NMS + matching + append, from the first loss kernel on).  The card's name, power limit and SM clock limit
are read in the same run and printed with the numbers.

    python tools/exp_val_time.py [--models v8n,v11s] [--batch 32] [--reps 10]"""
import argparse
import ctypes as C
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.exp_eval_time import card, kernels, time_ms  # noqa: E402


def run(model, B, reps):
    from tests.test_train_step import _targets
    from tests.util import oracle_model
    from yolosharp_b200 import _lib as L
    from yolosharp_b200.train_native import NativeTrainer
    arch, size = model[:-1], model[-1]
    tr = NativeTrainer(oracle_model(arch, "detect", size).state_dict(), arch, size, 80, device="cuda", max_batch=B, height=640, width=640)
    g = torch.Generator().manual_seed(0)
    x = torch.randint(0, 256, (B, 3, 640, 640), dtype=torch.uint8, generator=g).cuda()
    tg = _targets(B).contiguous()
    lib, sp = L.lib(), C.c_void_p(torch.cuda.current_stream().cuda_stream)
    calls = 2 * reps + 8
    L.check(lib.yb_trainer_val_begin(tr._h, calls * B, calls * tg.shape[0], sp))
    vb = lambda: L.check(lib.yb_trainer_val_batch(tr._h, C.c_void_p(x.data_ptr()), L.YB_U8, B, C.c_void_p(tg.data_ptr()), tg.shape[0], sp))
    ev = lambda: tr.evaluate(x)
    for _ in range(3):  # warm-up of every shape both paths launch
        ev(), vb()
    torch.cuda.synchronize()
    tv, te = [], []
    for _ in range(reps):  # alternated
        tv += time_ms(vb, 1)
        te += time_ms(ev, 1)
    tv, te = sorted(tv), sorted(te)
    med = lambda v: v[len(v) // 2]
    kv = kernels(vb)
    first_loss = next(i for i, k in enumerate(kv) if "loss_decode_kernel" in k[0])
    span = kv[-1][2] - kv[0][1]
    post = kv[-1][2] - kv[first_loss][1]
    items, metrics, counts = torch.empty(3), torch.empty(4), torch.zeros(3, dtype=torch.int32)
    L.check(lib.yb_trainer_val_end(tr._h, *(C.c_void_p(v.data_ptr()) for v in (items, metrics, counts)), sp))
    tr.close()
    return {"model": model, "batch": B, "val_batch_ms_median": round(med(tv), 3), "val_batch_ms_min": round(tv[0], 3),
            "evaluate_ms_median": round(med(te), 3), "evaluate_ms_min": round(te[0], 3),
            "val_batch_over_evaluate": round(med(tv) / med(te), 3), "detection_rows_per_image": round(int(counts[2]) / int(counts[0]), 1),
            "profiled": {"val_batch_span_ms": round(span / 1e3, 3), "post_forward_span_ms": round(post / 1e3, 3),
                         "post_forward_share": round(post / span, 3), "val_batch_kernels": len(kv),
                         "post_forward_kernels": len(kv) - first_loss}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="v8n,v11s")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("exp_val_time.py needs a GPU")
    print(json.dumps({"card": card(), "results": [run(m, a.batch, a.reps) for m in a.models.split(",")]}))


if __name__ == "__main__":
    main()
