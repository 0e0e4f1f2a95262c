"""pdt.nn.CrossEntropyLoss with probability targets it does not run natively, on the CPU: torch's result."""
import torch
import torch.nn.functional as F

import pytorch_distributed_train_b200 as pdt


def test_unbatched_probability_target_reaches_torch():
    """An unbatched [C] input with a [C] probability target, which torch's criterion accepts, gets torch's loss."""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(10, generator=g)
    q = torch.softmax(torch.randn(10, generator=g), 0)
    for kw in ({}, {"label_smoothing": 0.1}, {"reduction": "sum"}):
        crit = pdt.nn.CrossEntropyLoss(**kw)
        assert not crit.native_ok(x, q)
        assert torch.equal(crit(x, q), F.cross_entropy(x, q, **kw))
