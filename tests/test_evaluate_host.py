"""Host-side checks of NativeTrainer.evaluate that need no device: argument validation on a layout-only (DRY_RUN) trainer,
and the C entry point's refusals before any device work."""
import ctypes as C

import pytest
import torch


def _dry(max_batch=2, hw=64):
    from yolosharp_b200.train_native import NativeTrainer
    return NativeTrainer(None, "v8", "n", 80, device="cpu", max_batch=max_batch, height=hw, width=hw)


def test_evaluate_validates_images_before_any_device_call(built_lib):
    tr = _dry()
    with pytest.raises(ValueError, match="max_batch|takes 1..2"):
        tr.evaluate(torch.zeros(3, 3, 64, 64, dtype=torch.uint8))
    with pytest.raises(ValueError, match="takes"):
        tr.evaluate(torch.zeros(1, 3, 32, 64, dtype=torch.uint8))
    with pytest.raises(ValueError, match="uint8 or float32"):
        tr.evaluate(torch.zeros(1, 3, 64, 64, dtype=torch.float16))
    with pytest.raises(RuntimeError, match="without a device"):
        tr.evaluate(torch.zeros(1, 3, 64, 64, dtype=torch.uint8))
    tr.close()


def test_evaluate_entry_refuses_unbound_trainer(built_lib):
    from yolosharp_b200 import _lib as L
    tr = _dry()
    img = torch.zeros(1, 3, 64, 64, dtype=torch.uint8)
    lib = L.lib()
    assert lib.yb_trainer_evaluate(None, C.c_void_p(img.data_ptr()), L.YB_U8, 1, None, None, None, None) == -1
    assert lib.yb_trainer_evaluate(tr._h, C.c_void_p(img.data_ptr()), L.YB_U8, 1, None, None, None, None) == -4  # YB_ERR_STATE
    assert "yb_trainer_bind" in lib.yb_last_error().decode()
    tr.close()
