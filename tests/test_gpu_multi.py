"""Multi-GPU tests (need >= 2 H100s on one node; skipped otherwise - run with `python -m pytest
tests/test_gpu_multi.py -m gpu`): the library's peer-memory detection exchange (csrc/comm.cu, K12) and the sharded
predict call, one process per GPU."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _need(n):
    if not torch.cuda.is_available() or torch.cuda.device_count() < n:
        pytest.skip(f"needs {n} GPUs")


def _run(worker, world, *args):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=worker, args=(r, world, port, q) + args) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=600) for _ in range(world)]
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    return sorted(res)


def _init(rank, world, port):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))


def _comm_worker(rank, world, port, q, mode):
    _init(rank, world, port)
    try:
        from yolosharp_b200 import dist as ydist
        dev = torch.device("cuda", rank)
        B, MD, ROW = 4, 300, 6
        g = ydist.DetectionGather(B, MD, ROW, dev, mode=mode, slots=2)
        s = torch.cuda.Stream(dev)
        ok = True
        for step in range(12):  # several uses of both slots: exercises the sequence flags and the release / ack path
            slot = step & 1
            d, c = g.local_buffers(slot)
            with torch.cuda.stream(s):
                d.copy_(torch.full((B, MD, ROW), float(1000 * step + rank), device=dev) +
                        torch.arange(B * MD * ROW, device=dev).view(B, MD, ROW) * 1e-3)
                c.copy_(torch.arange(B, device=dev, dtype=torch.int32) + 100 * rank + step)
                g.gather(slot, stream=s)
                gd, gc = g.gathered(slot)
                gd, gc = gd.clone(), gc.clone()
            s.synchronize()
            for r in range(world):
                exp_d = torch.full((B, MD, ROW), float(1000 * step + r), device=dev) + \
                    torch.arange(B * MD * ROW, device=dev).view(B, MD, ROW) * 1e-3
                exp_c = torch.arange(B, device=dev, dtype=torch.int32) + 100 * r + step
                ok = ok and torch.equal(gd[r * B:(r + 1) * B], exp_d) and torch.equal(gc[r * B:(r + 1) * B], exp_c)
        torch.cuda.synchronize()
        dist.barrier()
        g.close()
        q.put((rank, bool(ok)))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("mode", ["comm", "nccl"])
def test_detection_gather_world2(mode):
    _need(2)
    assert _run(_comm_worker, 2, mode) == [(0, True), (1, True)]


def _predict_worker(rank, world, port, q):
    _init(rank, world, port)
    try:
        import yolosharp_b200 as y
        from yolosharp_b200 import dist as ydist
        from tests.util import oracle_model, synth_image
        dev = torch.device("cuda", rank)
        B = 3
        m = oracle_model("v8", "detect", "n")
        e = y.Engine("v8", "n", "detect", 80, "f16", rank, B, 320, 320)
        e.load_state_dict(m.state_dict())
        e.finalize()
        g = ydist.DetectionGather(B, 300, 6, dev, mode="comm", slots=2)
        shards = [[synth_image(B, 320, 320, seed=60 + 10 * it + r, dtype=torch.uint8).pin_memory() for r in range(world)]
                  for it in range(3)]
        dh = [torch.empty((world * B, 300, 6), dtype=torch.float32).pin_memory() for _ in range(2)]
        ch = [torch.empty((world * B,), dtype=torch.int32).pin_memory() for _ in range(2)]
        ok = True
        for rep in range(2):
            for it in range(3):
                slot = it & 1
                g.predict_submit(e, slot, shards[it][rank], dh[slot], ch[slot], 0.25, 0.45)
                g.predict_wait(e, slot)
                for r in range(world):  # every rank checks every shard against its own single-GPU predict of that shard
                    rd, rc = e.predict_u8(shards[it][r], 0.25, 0.45, 300)
                    ok = ok and torch.equal(ch[slot][r * B:(r + 1) * B], rc) and torch.equal(dh[slot][r * B:(r + 1) * B], rd)
                dist.barrier()
        torch.cuda.synchronize()
        dist.barrier()
        g.close()
        q.put((rank, bool(ok)))
    finally:
        dist.destroy_process_group()


def test_sharded_predict_gathers_all_ranks_world2():
    """yb_predict_u8_submit_gather on 2 GPUs: the host buffers of EVERY rank hold the detections of both shards in
    global image order, bit-identical to single-GPU predicts of the same shards (BASELINE configs[2] mechanics)."""
    _need(2)
    assert _run(_predict_worker, 2) == [(0, True), (1, True)]


def _train_worker(rank, world, port, q):
    _init(rank, world, port)
    try:
        from yolosharp_b200.train_native import NativeTrainer
        from tests.test_train_step import _targets
        from tests.util import oracle_model, synth_image
        torch.manual_seed(0)
        sd = {k: v.detach().clone() for k, v in oracle_model("v8", "detect", "n").state_dict().items()}
        B, H, W = 2, 64, 96
        shards = [(synth_image(B, H, W, seed=70 + r).cuda(), _targets(B, seed=r)) for r in range(world)]
        mk = lambda: NativeTrainer(sd, "v8", "n", 80, device=torch.device("cuda", rank), max_batch=B, height=H, width=W, lr=1e-3)
        # what every rank should hold after the all-reduce: the sum of the per-shard gradients, each taken on its own
        want = None
        for x, t in shards:
            solo = mk()
            solo.group = False  # no collective
            solo.step(x, t)
            want = solo.grad.clone() if want is None else want + solo.grad
        ddp = mk()
        ddp.step(*shards[rank])
        torch.cuda.synchronize()
        scale = float(want.abs().max())
        err = float((ddp.grad - want).abs().max()) / scale
        # the updated weights must be the same on every rank (same summed gradient, same AdamW)
        w = [torch.empty_like(ddp.flat) for _ in range(world)]
        dist.all_gather(w, ddp.flat)
        same = all(torch.equal(w[0], wi) for wi in w)
        q.put((rank, err < 1e-6, same))
    finally:
        dist.destroy_process_group()


def _two_devices_worker(q):
    try:
        import yolosharp_b200 as y
        from yolosharp_b200.engine import nms
        from yolosharp_b200.train_native import NativeTrainer
        from tests.test_train_step import _targets
        from tests.util import oracle_model, synth_image
        det_sd = oracle_model("v8", "detect", "n").state_dict()
        train_sd = {k: v.detach().clone() for k, v in oracle_model("v11", "detect", "n").state_dict().items()}
        x, xt, t = synth_image(2, 640, 640, seed=3), synth_image(2, 128, 128, seed=4), _targets(2)
        res = []
        for d in (0, 1):
            with torch.cuda.device(d):
                e = y.Engine("v8", "n", "detect", 80, "f16", d, 2, 640, 640)
                e.load_state_dict(det_sd)
                e.finalize()
                dets, counts, _ = nms(e.forward(x.cuda(d)))
                tr = NativeTrainer(train_sd, "v11", "n", 80, device=torch.device("cuda", d), max_batch=2, height=128, width=128,
                                   lr=1e-3)
                items = tr.step(xt.cuda(d), t)
                torch.cuda.synchronize()
                res.append({"dets": dets.cpu(), "counts": counts.cpu(), "loss items": items.clone(), "grad": tr.grad.cpu()})
                tr.close()
                e.close()
        # the loss items are summed over blocks with float atomics, so two runs on one device may differ in the last bit;
        # the gradient does not depend on them and must match exactly
        a, b = res
        q.put([k for k in a if not (torch.allclose(a[k], b[k], rtol=1e-6, atol=0) if k == "loss items" else torch.equal(a[k], b[k]))])
    except Exception as ex:  # a refused launch surfaces as YbError from the call that made it
        q.put(repr(ex))


def test_two_devices_in_one_process():
    """An f16 engine (forward + NMS) and a v11n native training step on device 0, then the same on device 1, in one fresh
    process: every kernel that needs more than 48 KiB of shared memory must get its limit on the second device too (the
    limit is a per-device function attribute), and device 1 must reproduce device 0 bit for bit."""
    _need(2)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    p = ctx.Process(target=_two_devices_worker, args=(q,))
    p.start()
    res = q.get(timeout=600)
    p.join(120)
    assert res == [], res
    assert p.exitcode == 0


def test_native_train_step_allreduce_world2():
    """The native step on 2 GPUs (BASELINE configs[3] mechanics): after yb_train_backward + the NCCL all-reduce of the flat
    gradient buffer every rank holds the SUM of the two shards' gradients (each equal to a single-GPU step on that shard:
    BatchNorm statistics stay per rank, as DDP without SyncBN), and yb_train_apply leaves identical weights on both ranks."""
    _need(2)
    assert _run(_train_worker, 2) == [(0, True, True), (1, True, True)]
