"""PDT_CONV_IMPL cannot pick another per-op conv2 kernel: conv2 always runs the TMA-im2col kernels, and a value naming another
kernel (bench.py --conv-impl simt|tcgen05) is refused before any tensor or device is touched, never silently ignored."""
import pytest
import torch
import torch.nn as nn

from pytorch_distributed_train_b200 import ops
from pytorch_distributed_train_b200.ops import functional


def _layer():
    return torch.rand(2, 16, 14, 14), nn.Conv2d(16, 32, 5, padding=2), nn.BatchNorm2d(32)


@pytest.mark.parametrize("value", ["simt", "tcgen05", "win"])
def test_conv_impl_naming_another_kernel_is_refused(monkeypatch, value):
    monkeypatch.setenv("PDT_CONV_IMPL", value)

    def reached(*args):
        raise AssertionError("the per-op convolution ran")

    monkeypatch.setattr(functional._ConvBnReluPool, "apply", reached)
    with pytest.raises(ValueError, match="TMA-im2col") as e:
        ops.conv_bn_relu_pool(*_layer())
    assert repr(value) in str(e.value)


@pytest.mark.parametrize("value", [None, "auto", "tma"])
def test_conv_impl_default_values_reach_the_kernels(monkeypatch, value):
    if value is None:
        monkeypatch.delenv("PDT_CONV_IMPL", raising=False)
    else:
        monkeypatch.setenv("PDT_CONV_IMPL", value)
    monkeypatch.setattr(functional._ConvBnReluPool, "apply", lambda *args: "reached")
    assert ops.conv_bn_relu_pool(*_layer()) == "reached"
