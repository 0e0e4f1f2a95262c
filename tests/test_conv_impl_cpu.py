"""The `impl` selector of the per-op convolution bindings is checked before anything touches a tensor or a device:
an unknown kernel family is an error that names the accepted values, never a silent fall-back to another kernel."""
import pytest
import torch

from pytorch_distributed_train_b200 import _C


def test_unknown_conv_impl_is_rejected():
    x = torch.zeros(1, 14, 14, 16)
    dy = torch.zeros(1, 14, 14, 32)
    w = torch.zeros(32, 16, 5, 5)
    for call in (lambda: _C.conv5x5_fwd(x, w, None, False, "win"),
                 lambda: _C.conv5x5_dgrad(dy, w, "win"),
                 lambda: _C.conv5x5_wgrad(dy, x, torch.zeros_like(w), None, "win")):
        with pytest.raises(RuntimeError, match="auto, tma, tcgen05, simt") as e:
            call()
        assert "'win'" in str(e.value)
