"""Which ConvNets the fused kernels take.  The two fused backward kernels write all ten parameter gradients and stage the classifier
weights in 16-byte copies, so a partially trainable model (a frozen layer) or a classifier weight that is not 16-byte aligned (a
user-made view: DDP's gradient arenas align every parameter) runs on the per-op kernels, whose gradients match float64 at the
tolerances of test_kernel_edges.py."""
import pytest
import torch
import torch.nn.functional as F

import pytorch_distributed_train_b200 as pdt
from pytorch_distributed_train_b200.ops import functional as OF

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _fp32_reference():
    # the oracle must be true fp32: no TF32 inside cuDNN/cuBLAS
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def dev():
    return torch.device("cuda", 0)


def _misalign_fc_weight(net):
    """Replace fc.weight by a parameter with the same values that starts 4 bytes into its storage."""
    w = net.fc.weight.detach()
    buf = torch.empty(w.numel() + 1, device=w.device)
    view = buf[1:].view_as(w)
    view.copy_(w)
    net.fc.weight = torch.nn.Parameter(view)
    assert net.fc.weight.data_ptr() % 16 != 0 and net.fc.weight.is_contiguous()


@pytest.mark.parametrize("case", ["frozen_conv1", "frozen_fc", "misaligned_fc_weight"])
def test_partially_trainable_convnet_takes_the_per_op_kernels(case):
    torch.manual_seed(1)
    net = pdt.models.ConvNet(fused=True).to(dev())
    ref = pdt.models.ConvNet(fused=False).to(dev())
    ref.load_state_dict(net.state_dict())
    ref = ref.double()
    x = torch.rand(100, 1, 28, 28, device=dev())
    t = torch.randint(0, 10, (100,), device=dev())
    assert OF.fused_convnet_ok(x, net)
    if case == "frozen_conv1":
        net.layer1[0].requires_grad_(False)
    elif case == "frozen_fc":
        net.fc.requires_grad_(False)
    else:
        _misalign_fc_weight(net)
    assert not OF.fused_convnet_ok(x, net)
    loss = pdt.nn.CrossEntropyLoss()(net(x), t)
    loss.backward()
    ref_loss = F.cross_entropy(ref(x.double()), t)
    ref_loss.backward()
    # conv2 runs in TF32 (10-bit mantissa) forward and in dgrad: ~1e-3 relative per product
    assert abs(loss.item() - ref_loss.item()) < 2e-3, (loss.item(), ref_loss.item())
    for (n1, p1), (_, p2) in zip(net.named_parameters(), ref.named_parameters()):
        if not p1.requires_grad:
            assert p1.grad is None, n1
            continue
        # TF32 as above, measured over the whole tensor; conv biases in front of a BatchNorm have a true gradient of zero (noise level)
        err, norm = (p1.grad.double() - p2.grad).norm().item(), p2.grad.norm().item()
        assert err <= 3e-2 * norm + 1e-4 * p2.numel() ** 0.5, (n1, err, norm)
