"""Elastic deformation of a batch, every image with its own displacement field: torchvision's ``transforms.v2.ElasticTransform``
definition (Simard, Steinkraus & Platt, ICDAR 2003), drawn, blurred and applied on the device in one launch (``ops.elastic``), so
that it can run inside a captured training step (``engine.GraphedTrainStep(augment=...)``)."""
from __future__ import annotations

import math
import numbers
from collections.abc import Sequence
from typing import Optional

import torch
import torch.nn.functional as F

from .augment import _sample_cpu


def _setup_number_or_seq(arg, name):
    """torchvision's ``_setup_number_or_seq``: a number or a sequence of one or two numbers → [float, float]."""
    if not isinstance(arg, (int, float, Sequence)):
        raise TypeError(f"{name} should be a number or a sequence of numbers. Got {type(arg)}")
    if isinstance(arg, Sequence) and len(arg) not in (1, 2):
        raise ValueError(f"If {name} is a sequence its length should be 1 or 2. Got {len(arg)}")
    if isinstance(arg, Sequence):
        for element in arg:
            if not isinstance(element, (int, float)):
                raise ValueError(f"{name} should be a sequence of numbers. Got {type(element)}")
        return [float(arg[0]), float(arg[-1])]
    return [float(arg), float(arg)]


def _gaussian_kernel1d(k: int, sigma: float) -> torch.Tensor:
    """torchvision's ``_get_gaussian_kernel1d`` in fp32 on the host: softmax(−(linspace(−lim, lim, k)/σ)²), lim = (k − 1)/(2√2)."""
    lim = (k - 1) / (2.0 * math.sqrt(2.0))
    x = torch.linspace(-lim, lim, steps=k, dtype=torch.float32)
    return torch.softmax(x.div(sigma).pow(2).neg(), dim=0)


class ElasticTransform:
    """Elastic deformation of every image of an fp32 ``[B, C, H, W]`` batch, each image with its own displacement field.  The
    arguments, their checks and their error messages are torchvision's ``v2.ElasticTransform`` (``fill`` is one number).  Per image,
    with torchvision's ``make_params`` and ``elastic``:

        dx0, dy0 ~ U[-1, 1) over H×W (torch.rand·2 − 1 in fp32, dx0 first);
        with sigma[0] > 0, dx0 is blurred by torchvision's ``gaussian_blur`` with kernel size kx = int(8·sigma[0] + 1) made odd and
        sigmas (sigma[0], sigma[1]), reflect-padded; dy0 likewise when sigma[1] > 0, with ky from sigma[1] and the same sigmas;
        dx = blurred_dx · alpha[0] / W,  dy = blurred_dy · alpha[1] / H  (fp32);

    output pixel (i, j) samples the image at (j + dx·W/2, i + dy·H/2) (``interpolation`` ``"nearest"`` or ``"bilinear"``, ``fill``
    where the source lies outside the image); all channels share the field.  torchvision's transform gives every image its own field
    only as a per-sample ``transform=``; called on a batch tensor it draws one field and warps the whole batch with it.

    * A CUDA batch takes the native kernel: one launch, the noise drawn on the device from ``generator`` (a CUDA generator on the
      batch's device; the default one when None), capturable in a CUDA graph where every replay draws new fields.
      ``torch.manual_seed`` (or the generator's ``manual_seed``) reproduces the sequence.  The blur weights are copied to the
      device by the first call there, so call the transform once before capturing it in a graph.
    * A CPU batch takes torch ops with the same definition, drawing image 0's dx0, its dy0, then image 1's ... from ``generator``
      (a CPU generator; torch's default one when None), as a loop of torchvision's transform over the images draws.
    * Any other dtype raises ``TypeError``.  As in torchvision, one positive and one non-positive sigma raise ``ValueError`` and a
      blur kernel whose half is not below the image's height and width raises ``RuntimeError``, both at call time.

    ``record_params=True`` keeps the last call's unblurred noise in ``last_params``: fp32 ``[B, 2, H, W]`` (dx0, dy0) on the batch's
    device, from which the field follows.  Inside a CUDA graph it is the graph's static tensor, holding the last replay's draws."""

    def __init__(self, alpha=50.0, sigma=5.0, interpolation="bilinear", fill: float = 0.0, generator: Optional[torch.Generator] = None,
                 record_params: bool = False):
        self.alpha = _setup_number_or_seq(alpha, "alpha")
        self.sigma = _setup_number_or_seq(sigma, "sigma")
        interpolation = getattr(interpolation, "value", interpolation)   # torchvision's InterpolationMode
        if interpolation not in ("nearest", "bilinear"):
            raise ValueError(f"Interpolation mode '{interpolation}' is unsupported with Tensor input")
        self.interpolation = interpolation
        if not isinstance(fill, numbers.Real):
            raise TypeError(f"fill should be a number, got {type(fill)}")
        self.fill = float(fill)
        self.generator = generator
        self.record_params = bool(record_params)
        self.last_params: Optional[torch.Tensor] = None
        # kernel sizes of the dx and dy blurs (0: none), and their 1-D weights: (kx, sigma[0]), (kx, sigma[1]), (ky, sigma[0]),
        # (ky, sigma[1]); kept on every device the transform has run on, for as long as the transform lives (a captured graph reads
        # them at every replay)
        self._ksizes = [self._ksize(s) if s > 0.0 else 0 for s in self.sigma]
        self._host_weights = (None if not any(self._ksizes) or min(self.sigma) <= 0.0 else
                              torch.cat([_gaussian_kernel1d(k, s) for k in self._ksizes for s in self.sigma]))
        self._device_weights: dict = {}

    @staticmethod
    def _ksize(sigma: float) -> int:
        k = int(8 * sigma + 1)
        return k + 1 if k % 2 == 0 else k

    def __repr__(self) -> str:
        return f"ElasticTransform(alpha={self.alpha}, sigma={self.sigma}, interpolation={self.interpolation!r}, fill={self.fill})"

    def _check_blur(self, H: int, W: int) -> None:
        """torchvision's errors for this size, in the order its make_params meets them."""
        for k in self._ksizes:
            if k == 0:
                continue
            if min(self.sigma) <= 0.0:
                raise ValueError(f"sigma should have positive values. Got {self.sigma}")
            pad = k // 2
            for arg, dim, size in ((4, 3, W), (6, 2, H)):
                if pad >= size:
                    raise RuntimeError(f"Argument #{arg}: Padding size should be less than the corresponding input dimension, but got: "
                                       f"padding ({pad}, {pad}) at dimension {dim} of input [1, 1, {H}, {W}]")

    def __call__(self, images: torch.Tensor) -> torch.Tensor:
        if images.dtype != torch.float32:
            raise TypeError(f"ElasticTransform: images must be float32 (got {images.dtype})")
        if images.dim() != 4:
            raise ValueError(f"ElasticTransform: images must be [B, C, H, W] (got shape {tuple(images.shape)})")
        H, W = images.shape[2:]
        self._check_blur(H, W)
        bilinear = self.interpolation == "bilinear"
        if images.is_cuda:
            from .. import ops

            weights = None
            if self._host_weights is not None:
                index = images.device.index if images.device.index is not None else torch.cuda.current_device()
                weights = self._device_weights.get(index)
                if weights is None:
                    if torch.cuda.is_current_stream_capturing():
                        raise RuntimeError("ElasticTransform: call the transform once on this device before capturing it in a CUDA "
                                           "graph; its first call there copies the blur weights to the device")
                    weights = self._device_weights[index] = self._host_weights.to(images.device)
            out, noise = ops.elastic(images.contiguous(), weights, self._ksizes, self.alpha, bilinear=bilinear, fill=self.fill,
                                     generator=self.generator, record_params=self.record_params)
        else:
            out, noise = _elastic_cpu(images, self.alpha, self._ksizes, self.sigma, bilinear, self.fill, self.generator)
        if self.record_params:
            self.last_params = noise
        return out


def _elastic_cpu(x, alpha, ksizes, sigma, bilinear, fill, generator):
    """The CPU path of ElasticTransform: torchvision's draws, blur and scaling in torch ops, the warp with coordinates in float64."""
    B, C, H, W = x.shape
    noise = torch.empty(B, 2, H, W)
    for b in range(B):
        for c in range(2):
            noise[b, c] = torch.rand(H, W, generator=generator) * 2 - 1
    if B == 0:
        return x.clone(), noise
    disp = []
    for c, (k, a, size) in enumerate(zip(ksizes, alpha, (W, H))):
        d = noise[:, c:c + 1]
        if k:
            # torchvision's gaussian_blur: the outer product of the y and x weights over the reflect-padded plane
            kernel = _gaussian_kernel1d(k, sigma[1]).unsqueeze(-1) * _gaussian_kernel1d(k, sigma[0])
            d = F.conv2d(F.pad(d, [k // 2] * 4, mode="reflect"), kernel.view(1, 1, k, k))
        disp.append((d * a / size).view(B, H, W))
    src_x = torch.arange(W, dtype=torch.float64).view(1, 1, W) + disp[0].double() * (0.5 * W)
    src_y = torch.arange(H, dtype=torch.float64).view(1, H, 1) + disp[1].double() * (0.5 * H)
    return _sample_cpu(x, src_x, src_y, bilinear, fill), noise
