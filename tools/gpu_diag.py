"""First-contact diagnostics on a real H100 (not a test: prints per-op errors, never asserts).
Each section runs in its own subprocess so that a trapped kernel (sticky CUDA error) cannot take
the other sections down.   python tools/gpu_diag.py [section ...]"""
import os
import subprocess
import sys
import time
import traceback

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def per_op_report(e, model, x_cpu, x_dev, tag, ref_engine=None, show=400):
    import torch
    from tests.util import expected_for_op, oracle_activations, rel_err
    (inf, _), acts = oracle_activations(model, x_cpu)
    pred = e.forward(x_dev)
    torch.cuda.synchronize()
    B = x_cpu.shape[0]
    worst = 0.0
    if ref_engine is not None:
        ref_engine.forward(x_dev)
        torch.cuda.synchronize()
    for i, name in enumerate(e.op_names()):
        exp = expected_for_op(model, acts, name)
        if exp is None:
            continue
        try:
            got = e.read_activation(i, B)
        except Exception as ex:
            print(f"[{tag}] {i:3d} {name:28s} not materialised ({str(ex)[-40:]})")
            continue
        if tuple(got.shape) != tuple(exp.shape):
            print(f"[{tag}] {i:3d} {name:28s} SHAPE got {tuple(got.shape)} exp {tuple(exp.shape)}")
            continue
        err = rel_err(got, exp)
        extra = ""
        if ref_engine is not None:
            extra = f" vs_ref_engine {rel_err(got, ref_engine.read_activation(i, B)):.3e}"
        worst = max(worst, err)
        flag = "  <<<<" if not (err < 0.05) else ""
        if i < show:
            print(f"[{tag}] {i:3d} {name:28s} {str(tuple(exp.shape)):22s} rel_err {err:.3e}{extra}{flag}")
    pe = (pred.cpu() - inf["boxes"]).abs()
    print(f"[{tag}] pred max abs err boxes {float(pe[:, :4].max()):.4e} scores {float(pe[:, 4:].max()):.4e} "
          f"worst op rel_err {worst:.3e}")
    return pred


def sec_fp32():
    import torch
    import yolosharp_b200 as y
    from tests.util import oracle_model, synth_image
    m = oracle_model("v8", "detect", "n")
    x = synth_image(2, 256, 320)
    e = y.Engine("v8", "n", "detect", 80, "f32", 0, 2, 256, 320, flags=2)
    e.load_state_dict(m.state_dict())
    e.finalize()
    per_op_report(e, m, x, x.cuda(), "fp32")


def sec_nms():
    import numpy as np
    import torch
    import yolosharp_b200 as y
    from tests.util import golden_nms_cases
    for tag, pred, nc, conf, iou, counts, rows, keep in golden_nms_cases():
        dets, cnt, kidx = y.nms(pred.cuda(), conf, iou, 300, nc)
        torch.cuda.synchronize()
        cnt = cnt.cpu().numpy()
        got_rows = np.concatenate([dets[i, :cnt[i]].cpu().numpy() for i in range(len(cnt))], 0)
        got_keep = np.concatenate([kidx[i, :cnt[i]].cpu().numpy() for i in range(len(cnt))], 0)
        ok_c = cnt.tolist() == counts.tolist()
        ok_r = got_rows.shape == rows.shape and np.array_equal(got_rows, rows)
        ok_k = got_keep.shape == keep.shape and np.array_equal(got_keep, keep)
        print(f"[nms] {tag:22s} counts {cnt.tolist()} exp {counts.tolist()} rows_exact {ok_r} keep_exact {ok_k}")
        if ok_c and not ok_k:
            bad = np.nonzero(got_keep != keep)[0]
            print("      first mismatches at", bad[:10], got_keep[bad[:5]], keep[bad[:5]])


def sec_f16gen():
    import yolosharp_b200 as y
    from tests.util import oracle_model, synth_image
    m = oracle_model("v8", "detect", "n")
    x = synth_image(2, 256, 320)
    e = y.Engine("v8", "n", "detect", 80, "f16", 0, 2, 256, 320, flags=3)
    e.load_state_dict(m.state_dict())
    e.finalize()
    per_op_report(e, m, x, x.cuda(), "f16-generic")


def sec_f16tc():
    import yolosharp_b200 as y
    from tests.util import oracle_model, synth_image
    m = oracle_model("v8", "detect", "n")
    x = synth_image(2, 256, 320)
    ref = y.Engine("v8", "n", "detect", 80, "f16", 0, 2, 256, 320, flags=3)
    ref.load_state_dict(m.state_dict())
    ref.finalize()
    e = y.Engine("v8", "n", "detect", 80, "f16", 0, 2, 256, 320, flags=2)
    e.load_state_dict(m.state_dict())
    e.finalize()
    per_op_report(e, m, x, x.cuda(), "f16-tc", ref_engine=ref)


def sec_f16tc_s():
    """v8s widths exercise BK=32/64 slabs and wider N tiles."""
    import yolosharp_b200 as y
    from tests.util import oracle_model, synth_image
    m = oracle_model("v8", "detect", "s")
    x = synth_image(1, 256, 320)
    ref = y.Engine("v8", "s", "detect", 80, "f16", 0, 1, 256, 320, flags=3)
    ref.load_state_dict(m.state_dict())
    ref.finalize()
    e = y.Engine("v8", "s", "detect", 80, "f16", 0, 1, 256, 320, flags=2)
    e.load_state_dict(m.state_dict())
    e.finalize()
    per_op_report(e, m, x, x.cuda(), "f16-tc-s", ref_engine=ref)


def sec_time():
    import torch
    import yolosharp_b200 as y
    from tests.util import oracle_model, synth_image
    for size, B in (("n", 32), ("s", 32), ("x", 8)):
        m = oracle_model("v8", "detect", size)
        for prec, flags in (("f16", 0), ("f16", 1), ("f32", 0)):
            if size != "n" and flags == 1:
                continue
            e = y.Engine("v8", size, "detect", 80, prec, 0, B, 640, 640, flags=flags)
            e.load_state_dict(m.state_dict())
            e.finalize()
            x = synth_image(B, 640, 640, dtype=torch.float16 if prec == "f16" else torch.float32).cuda()
            pred = torch.empty((B, 84, 8400), device="cuda")
            for _ in range(3):
                e.forward(x, pred)
            torch.cuda.synchronize()
            t0 = torch.cuda.Event(enable_timing=True)
            t1 = torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(10):
                e.forward(x, pred)
            t1.record()
            torch.cuda.synchronize()
            ms = t0.elapsed_time(t1) / 10
            print(f"[time] v8{size} B={B} {prec} flags={flags}: {ms:.3f} ms/forward  {B / ms * 1000:.0f} img/s")
            e.close()


SECTIONS = {"fp32": sec_fp32, "nms": sec_nms, "f16gen": sec_f16gen, "f16tc": sec_f16tc, "f16tc_s": sec_f16tc_s,
            "time": sec_time}

if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "--run":
        try:
            SECTIONS[sys.argv[2]]()
        except Exception:
            traceback.print_exc()
            sys.exit(1)
        sys.exit(0)
    names = sys.argv[1:] or list(SECTIONS)
    for n in names:
        t = time.time()
        print(f"===== {n} =====", flush=True)
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--run", n], timeout=900)
        print(f"===== {n} exit {r.returncode} in {time.time() - t:.1f}s =====", flush=True)
